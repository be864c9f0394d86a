"""CPU tests of the launch plan of a float group (lpcnet_b200_debug_group_plan_float, host only).  The streams per CTA (spc) come
from the group plan of test_group_plan.py; the kernel is then chosen as for a float batch (launch_sample, batch_api.cu): the
neuron-per-lane kernel at spc <= 4 unless LPCNET_B200_FLOAT_LANE_STREAM is set, with S = 1, 2 or 4 streams laid out per CTA (spc 3
-> 4), and the lane == stream kernel with spc slots otherwise.  Member k takes ceil(n_k / slots) consecutive CTAs of its own."""
import math
import pytest
import lpcnet_b200
from lpcnet_b200 import api
from test_group_plan import CASES, SPC_MAX, reference_spc, slot_map

FN_S = 4


@pytest.fixture(scope="module")
def L():
    from lpcnet_b200 import build
    build.build()
    return lpcnet_b200


def expected(spc, lane_stream):
    """(kernel, slots) a float batch launches at `spc` streams per CTA"""
    if spc <= FN_S and not lane_stream:
        return "neuron", {1: 1, 2: 2, 3: 4, 4: 4}[spc]
    return "lane", spc


@pytest.mark.parametrize("lane_stream", [False, True])
@pytest.mark.parametrize("spc", range(1, SPC_MAX + 1))
def test_kernel_and_slots_at_every_spc(L, spc, lane_stream):
    sizes = [3, 40, 17, 1]
    kernel, got_spc, slots, ctas = api.group_plan_float(sizes, 132, spc, lane_stream)
    assert got_spc == spc
    assert (kernel, slots) == expected(spc, lane_stream)
    assert ctas == sum(math.ceil(n / slots) for n in sizes)


def test_spc_3_lays_out_4_streams(L):
    assert api.group_plan_float([12, 5], 132, 3) == ("neuron", 3, 4, 3 + 2)
    assert api.group_plan_float([12, 5], 132, 3, lane_stream=True) == ("lane", 3, 3, 4 + 2)


@pytest.mark.parametrize("sizes", [[1, 1], [64] * 4, [130, 2, 3], [7] * 16])
def test_lane_stream_forces_the_lane_kernel_at_small_spc(L, sizes):
    k0, spc0, _, _ = api.group_plan_float(sizes, 132)
    k1, spc1, slots1, ctas1 = api.group_plan_float(sizes, 132, lane_stream=True)
    assert spc0 == spc1 <= FN_S and k0 == "neuron" and k1 == "lane"
    assert slots1 == spc1 and ctas1 == sum(math.ceil(n / spc1) for n in sizes)


@pytest.mark.parametrize("lane_stream", [False, True])
@pytest.mark.parametrize("sms", [132, 133])
@pytest.mark.parametrize("sizes", CASES + [[32, 64, 128], [64] * 4, [1024] * 8, [33, 131, 264, 100]],
                         ids=lambda v: "-".join(map(str, v)))
def test_every_stream_in_one_live_slot_and_no_cta_mixes_members(L, sizes, sms, lane_stream):
    kernel, spc, slots, ctas = api.group_plan_float(sizes, sms, 0, lane_stream)
    assert spc == reference_spc(sizes, sms)                     # spc is the int8 group's plan, unchanged
    assert spc == api.group_plan(sizes, sms)[0]
    assert (kernel, slots) == expected(spc, lane_stream)
    assert ctas == sum(math.ceil(n / slots) for n in sizes)
    live, total = slot_map(sizes, slots)                         # CTA c of member k holds its streams c*slots .. c*slots + slots - 1
    assert total == ctas
    assert sorted(live.values()) == [(k, s) for k, n in enumerate(sizes) for s in range(n)]
    members = {}
    for (c, _), (k, _) in live.items():
        members.setdefault(c, set()).add(k)
    assert all(len(v) == 1 for v in members.values())
    assert sorted(members) == list(range(ctas))


@pytest.mark.parametrize("lane_stream", [False, True])
@pytest.mark.parametrize("override", [0, 1, 2, 3, 4, 5, 17, 32, 40])
@pytest.mark.parametrize("sms", [132, 133])
@pytest.mark.parametrize("n", [1, 2, 131, 132, 133, 263, 264, 265, 395, 396, 397, 527, 528, 529, 1024, 4224, 4225, 40000])
def test_one_member_plans_like_a_batch(L, n, sms, override, lane_stream):
    # a batch's plan (launch_sample, batch_api.cu) in closed form: min(32, max(1, override or ceil(n / SMs))); then its float kernel
    spc = min(SPC_MAX, max(1, override or math.ceil(n / sms)))
    small_float = spc <= FN_S and not lane_stream
    S = (1 if spc <= 1 else 2 if spc == 2 else FN_S) if small_float else spc
    assert api.group_plan_float([n], sms, override, lane_stream) == ("neuron" if small_float else "lane", spc, S, math.ceil(n / S))


def test_switch_points(L):
    """total streams around 132, 264 and 528 on 132 SMs: spc 1 -> 2 -> 3 (S 4) -> 4 -> 5 (lane == stream)"""
    assert api.group_plan_float([66, 66], 132)[:3] == ("neuron", 1, 1)
    assert api.group_plan_float([66, 67], 132)[:3] == ("neuron", 2, 2)
    assert api.group_plan_float([132, 132], 132)[:3] == ("neuron", 2, 2)
    assert api.group_plan_float([132, 133], 132)[:3] == ("neuron", 3, 4)
    assert api.group_plan_float([264, 264], 132)[:3] == ("neuron", 4, 4)
    assert api.group_plan_float([264, 265], 132)[:3] == ("lane", 5, 5)
    assert api.group_plan_float([2112, 2112], 132)[:3] == ("lane", 32, 32)
    assert api.group_plan_float([2112, 2113], 132) == ("lane", 32, 32, 66 + 67)       # past one wave


@pytest.mark.parametrize("sizes", [[], [0], [5, -1], [1] * 17])
def test_bad_plans_are_refused(L, sizes):
    with pytest.raises(api.LPCNetB200Error):
        api.group_plan_float(sizes, 132)


def test_bad_sms_is_refused(L):
    with pytest.raises(api.LPCNetB200Error):
        api.group_plan_float([4], 0)
