"""CPU tests of the launch plan of a group (lpcnet_b200_debug_group_plan, host only): one streams-per-CTA value (spc) for the
whole launch, the smallest for which the members' CTAs, ceil(n_k / spc) each, fit the SMs (32 when nothing fits), an override
pinning it, and member k on consecutive CTAs of its own.  The slot map below restates the kernel's (sample_kernel.cu
slot_stream): CTA c of member k holds the member's streams c*spc .. c*spc + spc - 1 that exist."""
import math
import pytest
import lpcnet_b200
from lpcnet_b200 import api

SPC_MAX = 32

CASES = [
    [1],
    [1, 1, 1],
    [1, 4096],
    [1024] * 4,
    [4096],
    [31, 33, 63, 65],
    [15, 16, 17, 32, 33],
    [4095, 1, 4097 - 1],
    [132 * 32 + 1],
    [2000, 3000, 5000],                  # past one wave at 32 streams per CTA
    [512] * 8,
    [7] * 16,
    [130, 2, 3],
]


@pytest.fixture(scope="module")
def L():
    from lpcnet_b200 import build
    build.build()
    return lpcnet_b200


def reference_spc(sizes, sms):
    for s in range(1, SPC_MAX + 1):
        if sum(math.ceil(n / s) for n in sizes) <= sms:
            return s
    return SPC_MAX


def slot_map(sizes, spc):
    """(cta, slot) -> (member, stream) of every live slot, with member k on CTAs [cta0_k, cta0_k + ceil(n_k / spc))"""
    live, cta0 = {}, 0
    for k, n in enumerate(sizes):
        for c in range(math.ceil(n / spc)):
            for j in range(spc):
                s = c * spc + j
                if s < n:
                    live[(cta0 + c, j)] = (k, s)
        cta0 += math.ceil(n / spc)
    return live, cta0


@pytest.mark.parametrize("sms", [132, 133])
@pytest.mark.parametrize("sizes", CASES, ids=lambda v: "-".join(map(str, v)))
def test_plan_is_smallest_fit(L, sizes, sms):
    spc, ctas = api.group_plan(sizes, sms)
    assert spc == reference_spc(sizes, sms)
    assert ctas == sum(math.ceil(n / spc) for n in sizes)
    fits = [s for s in range(1, SPC_MAX + 1) if sum(math.ceil(n / s) for n in sizes) <= sms]
    if fits:
        assert ctas <= sms and spc == min(fits)
        if spc > 1:
            assert sum(math.ceil(n / (spc - 1)) for n in sizes) > sms
    else:
        assert spc == SPC_MAX and ctas > sms       # more than one wave


@pytest.mark.parametrize("sms", [132, 133])
@pytest.mark.parametrize("sizes", CASES, ids=lambda v: "-".join(map(str, v)))
def test_every_stream_in_one_live_slot_and_no_cta_mixes_members(L, sizes, sms):
    spc, ctas = api.group_plan(sizes, sms)
    live, total = slot_map(sizes, spc)
    assert total == ctas
    got = sorted(live.values())
    assert got == [(k, s) for k, n in enumerate(sizes) for s in range(n)]      # each group stream exactly once
    members = {}
    for (c, _), (k, _) in live.items():
        members.setdefault(c, set()).add(k)
    assert all(len(v) == 1 for v in members.values())
    assert sorted(members) == list(range(ctas))                                # no CTA without a live slot


@pytest.mark.parametrize("override", [1, 5, 16, 17, 32, 40])
@pytest.mark.parametrize("sizes", [[1], [31, 33, 63, 65], [2000, 3000, 5000]], ids=lambda v: "-".join(map(str, v)))
def test_override_is_honoured(L, sizes, override):
    spc, ctas = api.group_plan(sizes, 132, override)
    assert spc == min(override, SPC_MAX)
    assert ctas == sum(math.ceil(n / spc) for n in sizes)


@pytest.mark.parametrize("sms", [132, 133])
@pytest.mark.parametrize("n", [1, 2, 131, 132, 133, 263, 264, 265, 1024, 4095, 4096, 4224, 4225, 4257, 40000])
def test_one_member_plans_like_a_batch(L, n, sms):
    # a batch's plan (launch_sample, batch_api.cu) in closed form: min(32, max(1, ceil(n / SMs)))
    spc, ctas = api.group_plan([n], sms)
    assert spc == min(SPC_MAX, max(1, math.ceil(n / sms)))
    assert ctas == math.ceil(n / spc)


@pytest.mark.parametrize("sizes", [[], [0], [5, -1], [1] * 17])
def test_bad_plans_are_refused(L, sizes):
    with pytest.raises(api.LPCNetB200Error):
        api.group_plan(sizes, 132)
