"""CPU tests of the launch plan of a mixed group (lpcnet_b200_debug_mixed_plan, host only).  Members are classed by (GRU_A size,
flavour) in order of first appearance.  One streams-per-CTA value (spc) serves every class: the one a group over all members would
plan, the smallest at which sum ceil(n_k / spc) fits the SMs (32 when nothing fits), or the pinned value.  Each class then takes
the CTAs its own group takes at that spc: int8 classes ceil(n_k / spc) per member, float classes ceil(n_k / slots) with the kernel
and slots of a float group (neuron-per-lane with S = 1, 2 or 4 at spc <= 4 unless LPCNET_B200_FLOAT_LANE_STREAM, lane == stream
otherwise)."""
import math
import pytest
import lpcnet_b200
from lpcnet_b200 import api
from test_group_plan import SPC_MAX, reference_spc

FN_S = 4
SHAPES = [(na, fl) for fl in (0, 1) for na in (128, 256, 384)]


@pytest.fixture(scope="module")
def L():
    from lpcnet_b200 import build
    build.build()
    return lpcnet_b200


def float_kernel(spc, lane_stream):
    if spc <= FN_S and not lane_stream:
        return "neuron", {1: 1, 2: 2, 3: 4, 4: 4}[spc]
    return "lane", spc


def reference(sizes, shapes, sms, override=0, lane_stream=False):
    """(spc, class of each member, [(kernel, ctas)] per class) restated from the rules above"""
    spc = min(SPC_MAX, override) if override > 0 else reference_spc(sizes, sms)
    keys, cls, out = [], [], []
    for n, key in zip(sizes, shapes):
        if key not in keys:
            keys.append(key)
            out.append([float_kernel(spc, lane_stream)[0] if key[1] else "int8", 0])
        c = keys.index(key)
        cls.append(c)
        slots = float_kernel(spc, lane_stream)[1] if key[1] else spc
        out[c][1] += math.ceil(n / slots)
    return spc, cls, [tuple(v) for v in out]


def plan(sizes, shapes, sms, override=0, lane_stream=False):
    return api.mixed_plan(sizes, [s[0] for s in shapes], [s[1] for s in shapes], sms, override, lane_stream)


MIXES = [
    ([100, 200, 50], [(384, 0), (128, 0), (384, 1)]),
    ([1, 1], [(128, 0), (128, 1)]),
    ([64, 64, 64, 64], [(384, 0), (256, 0), (128, 0), (384, 0)]),
    ([1024, 256, 64], [(384, 0), (256, 0), (128, 0)]),
    ([2000, 3000, 5000], [(128, 1), (384, 0), (256, 1)]),            # past one wave at 32 streams per CTA
    ([7] * 16, [SHAPES[k % 6] for k in range(16)]),
    ([264, 265], [(384, 1), (384, 0)]),
    ([132, 133, 1], [(256, 1), (256, 1), (128, 0)]),
    ([33, 131, 264, 100, 5, 9], SHAPES),
]


@pytest.mark.parametrize("lane_stream", [False, True])
@pytest.mark.parametrize("sms", [132, 133])
@pytest.mark.parametrize("mix", MIXES, ids=lambda m: "-".join("%d:%d%s" % (n, s[0], "f" if s[1] else "") for n, s in zip(*m)))
def test_plan_matches_the_rules(L, mix, sms, lane_stream):
    sizes, shapes = mix
    assert plan(sizes, shapes, sms, 0, lane_stream) == reference(sizes, shapes, sms, 0, lane_stream)


@pytest.mark.parametrize("sms", [132, 133])
@pytest.mark.parametrize("mix", MIXES, ids=lambda m: "-".join(map(str, m[0])))
def test_spc_is_the_smallest_that_fits(L, mix, sms):
    """the classes' CTAs at spc fit the SMs together (counted ceil(n_k / spc) per member, and no more when a float class lays out
    more slots), and at spc - 1 they do not"""
    sizes, shapes = mix
    spc, _, classes = plan(sizes, shapes, sms)
    total = lambda s: sum(math.ceil(n / s) for n in sizes)
    if total(SPC_MAX) <= sms:
        assert total(spc) <= sms and sum(c for _, c in classes) <= total(spc)
        assert spc == 1 or total(spc - 1) > sms
    else:
        assert spc == SPC_MAX


def test_classes_in_order_of_first_appearance(L):
    shapes = [(128, 1), (384, 0), (128, 1), (256, 0), (384, 0), (128, 0), (256, 1), (384, 1), (256, 0)]
    _, cls, classes = plan([10] * len(shapes), shapes, 132)
    assert cls == [0, 1, 0, 2, 1, 3, 4, 5, 2]
    assert [k for k, _ in classes] == ["neuron", "int8", "int8", "int8", "neuron", "neuron"]


def test_flavour_splits_a_size(L):
    _, cls, classes = plan([5, 6], [(384, 0), (384, 1)], 132)
    assert cls == [0, 1] and len(classes) == 2


def test_one_class_for_one_shape(L):
    spc, cls, classes = plan([5, 6, 7], [(256, 0)] * 3, 132)
    assert cls == [0, 0, 0] and classes == [("int8", 18)] and spc == 1


# ---- a one-shape member list plans as its group, at every switch point ----
def switch_sizes(sms):
    """two members whose total is m * SMs and one more, for every spc switch 1..32, and past one wave"""
    out = []
    for m in range(1, SPC_MAX + 1):
        for extra in (0, 1):
            total = m * sms + extra
            a = m * (sms // 3)
            out.append([a, total - a])
    return out + [[1], [SPC_MAX * sms + 1]]


@pytest.mark.parametrize("na", [128, 256, 384])
@pytest.mark.parametrize("sms", [132, 133])
def test_one_int8_shape_plans_as_its_group(L, na, sms):
    for sizes in switch_sizes(sms):
        for override in (0, 5):
            spc, cls, classes = plan(sizes, [(na, 0)] * len(sizes), sms, override)
            g_spc, g_ctas = api.group_plan(sizes, sms, override)
            assert (spc, classes) == (g_spc, [("int8", g_ctas)]), sizes
            assert cls == [0] * len(sizes)


@pytest.mark.parametrize("lane_stream", [False, True])
@pytest.mark.parametrize("na", [128, 256, 384])
@pytest.mark.parametrize("sms", [132, 133])
def test_one_float_shape_plans_as_its_group(L, na, sms, lane_stream):
    for sizes in switch_sizes(sms):
        for override in (0, 3, 5):
            spc, _, classes = plan(sizes, [(na, 1)] * len(sizes), sms, override, lane_stream)
            kernel, g_spc, _, g_ctas = api.group_plan_float(sizes, sms, override, lane_stream)
            assert (spc, classes) == (g_spc, [(kernel, g_ctas)]), sizes


# ---- switches ----
@pytest.mark.parametrize("override", [1, 3, 4, 5, 16, 17, 32, 40])
def test_override_pins_spc(L, override):
    sizes, shapes = MIXES[0]
    spc, _, classes = plan(sizes, shapes, 132, override)
    assert spc == min(override, SPC_MAX)
    assert (spc, classes) == reference(sizes, shapes, 132, override)[::2]


@pytest.mark.parametrize("spc", [1, 2, 3, 4])
def test_lane_stream_switch_moves_float_classes_only(L, spc):
    sizes, shapes = [12, 12, 12], [(384, 0), (256, 1), (128, 1)]
    _, _, k0 = plan(sizes, shapes, 132, spc)
    _, _, k1 = plan(sizes, shapes, 132, spc, lane_stream=True)
    assert [k for k, _ in k0] == ["int8", "neuron", "neuron"]
    assert [k for k, _ in k1] == ["int8", "lane", "lane"]
    assert k0[0] == k1[0]
    assert [c for _, c in k1[1:]] == [math.ceil(12 / spc)] * 2


# ---- refusals ----
@pytest.mark.parametrize("sizes,shapes", [
    ([], []),
    ([0], [(384, 0)]),
    ([5, -1], [(384, 0), (128, 0)]),
    ([1] * 17, [(384, 0)] * 17),
    ([4], [(192, 0)]),
    ([4], [(512, 1)]),
    ([4], [(384, 2)]),
    ([4], [(384, -1)]),
])
def test_bad_plans_are_refused(L, sizes, shapes):
    with pytest.raises(api.LPCNetB200Error):
        plan(sizes, shapes, 132)


def test_bad_sms_and_lengths_are_refused(L):
    with pytest.raises(api.LPCNetB200Error):
        plan([4], [(384, 0)], 0)
    with pytest.raises(api.LPCNetB200Error):
        api.mixed_plan([4, 5], [384], [0, 0], 132)
