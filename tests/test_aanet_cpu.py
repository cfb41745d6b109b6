"""CPU: AANet -- the torchvision oracle of the modulated deformable convolution against a float64 evaluation of its formula, the
attribute set patch() installs on the reference's aanet, routing and refusals, and the envelope of DeformBottleneckEngine.serves()."""
import math

import pytest
import torch

from oracle import _reference_shim as shim
from oracle import aanet as oa

needs_model = pytest.mark.skipif(not shim.available() or not oa.extension_available(),
                                 reason="reference tree or its deform_conv_cuda build (oracle/_ref) not staged")


def _direct(x, off, mask, w, stride, pad, dil, dg):
    """out[b,o,y,x] = sum_{c,tap} W[o,c,tap] * m * bilinear(in[b,c], y*s - p + kh*d + dy, x*s - p + kw*d + dx), zero outside
    (-1, H) x (-1, W), each corner checked on its own -- written out in float64 loops."""
    b, cin, h, wd = x.shape
    cout = w.shape[0]
    ho, wo = off.shape[2:]
    cpg = cin // dg
    out = torch.zeros(b, cout, ho, wo, dtype=torch.float64)
    for n in range(b):
        for c in range(cin):
            g = c // cpg
            for tap in range(9):
                kh, kw = divmod(tap, 3)
                col = torch.zeros(ho, wo, dtype=torch.float64)
                for yo in range(ho):
                    for xo in range(wo):
                        hi = yo * stride - pad + kh * dil + float(off[n, g * 18 + 2 * tap, yo, xo])
                        wi = xo * stride - pad + kw * dil + float(off[n, g * 18 + 2 * tap + 1, yo, xo])
                        if not (hi > -1 and wi > -1 and hi < h and wi < wd):
                            continue
                        hl, wl = math.floor(hi), math.floor(wi)
                        lh, lw = hi - hl, wi - wl
                        v = 0.0
                        for yy, xx, wt in ((hl, wl, (1 - lh) * (1 - lw)), (hl, wl + 1, (1 - lh) * lw),
                                           (hl + 1, wl, lh * (1 - lw)), (hl + 1, wl + 1, lh * lw)):
                            if 0 <= yy < h and 0 <= xx < wd:
                                v += wt * float(x[n, c, yy, xx])
                        col[yo, xo] = v * float(mask[n, g * 9 + tap, yo, xo])
                out[n] += w[:, c, kh, kw].double().view(-1, 1, 1) * col
    return out


@pytest.mark.parametrize("stride,dil,dg,integer,from_logits", [(1, 1, 1, False, False), (1, 2, 2, True, True),
                                                                 (2, 1, 2, False, True), (2, 2, 1, True, False)])
def test_torchvision_oracle_equals_the_formula(stride, dil, dg, integer, from_logits):
    g = torch.Generator().manual_seed(stride * 10 + dil + dg)
    b, cin, cout, h, w = 2, 4, 3, 5, 7
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    x = torch.randn(b, cin, h, w, generator=g, dtype=torch.float64)
    off = torch.randn(b, dg * 18, ho, wo, generator=g, dtype=torch.float64) * 3
    if integer:
        off = off.round()
    off[0, 0, 0, 0], off[0, 1, 0, 1], off[-1, -2, -1, -1], off[-1, -1, -1, -2] = -50.0, 50.0, 40.0, -40.0   # beyond every edge
    m = torch.randn(b, dg * 9, ho, wo, generator=g, dtype=torch.float64)
    mask = 2 * torch.sigmoid(m) if from_logits else torch.rand(b, dg * 9, ho, wo, generator=g, dtype=torch.float64)
    wgt = torch.randn(cout, cin, 3, 3, generator=g, dtype=torch.float64)
    got = oa.modulated_deform_conv(x, off, mask, wgt, None, stride, dil, dil, dg)
    assert torch.allclose(got, _direct(x, off, mask, wgt, stride, dil, dil, dg), rtol=1e-10, atol=1e-10)


def _expected_overrides(m):
    # the refinements get a private copy of forward, the method that uses disp_warp (patch._rebind_methods); the deformable
    # bottlenecks keep the reference's extension (no override)
    return {"cost_volume", "disparity_estimation"} | {"refinement.%d" % i for i in range(len(m.refinement))}


@needs_model
def test_patch_surface_and_state_dict():
    from openstereo_b200.patch import patch
    m = oa.aanet()
    keys = list(m.state_dict())
    patch(m)
    assert list(m.state_dict()) == keys
    overridden = {name for name, mod in m.named_modules() if "forward" in vars(mod) and name}
    assert overridden == _expected_overrides(m)
    for ref in m.refinement:
        assert set(k for k in vars(ref) if not k.startswith("_") and k not in ("training",)) >= {"forward"}
        assert ref.forward.__func__.__globals__["disp_warp"] is not type(ref).forward.__globals__["disp_warp"]
    assert type(m.refinement[0]).forward.__globals__["disp_warp"].__module__.endswith("aanet.submodule")


@needs_model
def test_strict_refuses_cpu_and_non_strict_keeps_autograd():
    from openstereo_b200.patch import patch
    m = patch(oa.aanet())
    with pytest.raises(RuntimeError, match="CUDA inference only"):
        m.disparity_estimation(torch.randn(1, 16, 4, 8))
    with pytest.raises(RuntimeError, match="CUDA inference only"):
        m.cost_volume([torch.randn(1, 4, 4, 8)], [torch.randn(1, 4, 4, 8)])
    with pytest.raises(RuntimeError, match="CUDA inference only"):
        m.refinement[0].forward(torch.rand(1, 8, 16), torch.randn(1, 3, 8, 16), torch.randn(1, 3, 8, 16))
    lax = patch(oa.aanet(), strict=False).train()
    cost = torch.randn(1, 16, 4, 8, requires_grad=True)
    lax.disparity_estimation(cost).sum().backward()
    assert cost.grad is not None and cost.grad.abs().sum() > 0
    vol = lax.cost_volume([torch.randn(1, 4, 4, 8, requires_grad=True)], [torch.randn(1, 4, 4, 8)])
    assert vol[0].requires_grad


@needs_model
@pytest.mark.parametrize("kw", [dict(amp=True), dict(aggregation=True)])
def test_options_other_models_own_raise(kw):
    from openstereo_b200.patch import patch
    with pytest.raises(NotImplementedError):
        patch(oa.aanet(), **kw)


@needs_model
def test_routing_by_defining_module():
    from openstereo_b200.patch import _MODULE_PATCHERS, _PATCHERS, _patch_aanet
    assert _MODULE_PATCHERS[("aanet", "aanet", "aanet")] is _patch_aanet
    assert "aanet" not in _PATCHERS
    impostor = type("aanet", (torch.nn.Module,), {})()
    from openstereo_b200.patch import patch
    with pytest.raises(NotImplementedError):
        patch(impostor)


@needs_model
def test_engine_envelope():
    from openstereo_b200.aanet import DeformBottleneckEngine
    m = oa.aanet()
    blocks = [mod for mod in m.modules() if type(mod).__name__ in ("DeformBottleneck", "DeformSimpleBottleneck")]
    x = torch.zeros(1, 8, 4, 4)
    assert all(DeformBottleneckEngine(b).serves(x) for b in blocks)
    assert sorted({b.conv2.deform_conv.out_channels for b in blocks}) == [16, 32, 64, 128]
    blk = blocks[-1]
    assert not DeformBottleneckEngine(blk).serves(x.double())
    blk.conv2.modulation = False
    assert not DeformBottleneckEngine(blk).serves(x)
    blk.conv2.modulation = True
    blk.conv2.deform_conv.groups = 2
    assert not DeformBottleneckEngine(blk).serves(x)
    blk.conv2.deform_conv.groups = 1
    blk.conv2.double_mask = False
    assert not DeformBottleneckEngine(blk).serves(x)
