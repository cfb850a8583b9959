"""CPU tests of the inference-plan model in tests/infer_plan_ref.py, on unbound 16-bit inference plans (no GPU needed):
the topology against yb_net_layer_info / yb_net_layer_schedule, the `kernel` field of yb_net_layer_schedule under the
options that choose it, and that every configuration of tests/test_gpu_infer_plan.py reaches what it exists for."""
import ctypes as C

import pytest

from tests import infer_plan_ref as P


@pytest.fixture
def L():
    from yolov3_tensorflow_b200 import _lib
    P.set_options(_lib, {})
    yield _lib
    P.set_options(_lib, {})


def _plan(L, n, H, W, code):
    """(infos, schedules) of an unbound inference plan under the current options."""
    net = C.c_void_p()
    L.check(L.lib.yb_net_create(C.byref(net), P.CLASSES, n, H, W, code, 0), "net_create")
    try:
        infos = []
        for i in range(L.lib.yb_net_num_layers(net)):
            info = L.LayerInfo()
            L.check(L.lib.yb_net_layer_info(net, i, C.byref(info)), "layer_info")
            infos.append(info)
        return infos, P.layer_schedules(L, net)
    finally:
        L.lib.yb_net_destroy(net)


def test_topology_matches_inference_plan(L):
    topo = P.Topology()
    infos, scheds = _plan(L, 4, 416, 416, L.YB_F16)
    assert len(infos) == len(topo.table) == 75
    assert [i for i, s in enumerate(scheds) if s.residual] == topo.residual
    assert [f.index for f in infos if f.upsample2x] == topo.upsample
    assert [f.index for f in infos if not f.has_bn] == topo.heads
    # the concat buffers: [upsampled 256 | route 512] at 26^2 and [upsampled 128 | route 256] at 52^2
    assert (topo.out_ld[25], topo.out_off[25], topo.out_ld[67], topo.out_off[67]) == (384, 128, 384, 0)
    assert (topo.out_ld[42], topo.out_off[42], topo.out_ld[59], topo.out_off[59]) == (768, 256, 768, 0)
    assert topo.concat == {60: (59, 42), 68: (67, 25)}
    for i in range(1, 75):
        assert infos[i].cin == sum(infos[j].cout for j in topo.inputs[i]), i
        for j in topo.inputs[i]:
            up = 2 if infos[j].upsample2x else 1
            assert (infos[j].out_h * up, infos[j].out_w * up) == (infos[i].in_h, infos[i].in_w), (i, j)
    for b in topo.residual:                   # the shortcut out(b - 2) has the output's shape
        assert (infos[b - 2].out_h, infos[b - 2].out_w, infos[b - 2].cout) == (infos[b].out_h, infos[b].out_w, infos[b].cout)


@pytest.mark.parametrize("cid,opts,dt,weights,n,hw", P.CONFIGS, ids=[c[0] for c in P.CONFIGS])
def test_configuration_premise(L, cid, opts, dt, weights, n, hw):
    P.set_options(L, opts)
    code = L.YB_F16 if dt == "fp16" else L.YB_BF16
    infos, scheds = _plan(L, n, hw[0], hw[1], code)
    P.premise(cid, scheds, infos, P.Topology())


def test_kernel_field_follows_the_options(L):
    topo = P.Topology()
    c3 = topo.residual[0]
    IG, HALO, FUSED, STEM, THIN = L.YB_LAYER_IGEMM, L.YB_LAYER_HALO, L.YB_LAYER_FUSED_STEM, L.YB_LAYER_STEM, L.YB_LAYER_THIN

    def kernels(opts, code=L.YB_F16, hw=(416, 416)):
        P.set_options(L, opts)
        infos, scheds = _plan(L, 2, hw[0], hw[1], code)
        for i, s in enumerate(scheds):
            assert bool(s.igemm) == (s.kernel == IG), (opts, i, s.igemm, s.kernel)
        return infos, [s.kernel for s in scheds]

    infos, k = kernels({})
    assert k[:2] == [FUSED, FUSED] and k[c3] == HALO and k.count(HALO) == 1
    assert set(k[2:]) == {IG, HALO}
    _, k = kernels({}, code=L.YB_BF16)
    assert k[:2] == [FUSED, FUSED] and k[c3] == HALO
    _, k = kernels({"YB_STEM_FUSE": "0"})
    assert k[:2] == [STEM, HALO] and k[c3] == HALO
    _, k = kernels({"YB_HALO": "0"})
    assert HALO not in k and FUSED not in k and k[0] == STEM and set(k[1:]) == {IG}
    _, k = kernels({"YB_HALO": "1"})
    halo = [i for i in range(2, 75) if k[i] == HALO]
    assert k[:2] == [FUSED, FUSED] and c3 in halo and len(halo) > 1
    for i in halo:                            # only 3x3 convs with 32 / 64 input and 64 / 128 output channels
        assert infos[i].ksize == 3 and infos[i].cin in (32, 64) and infos[i].cout in (64, 128)
    _, k = kernels({"YB_THIN": "2"})
    assert k[0] == STEM and k[1] == THIN and k[c3] == THIN and k.count(THIN) == 2
    _, k = kernels({"YB_THIN": "0"})          # the CUDA-core stem switch leaves the fused stem alone
    assert k[:2] == [FUSED, FUSED]
