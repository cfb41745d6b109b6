"""CPU: MSNet3D -- the oracle against its fixtures and the live reference, use_res_connect of every block, the new C-ABI entry
point, and patch()'s drop-in contract on the unmodified reference class (no compute on a GPU here)."""
import pytest
import torch

from oracle import _reference_shim as shim
from oracle import msnet as oms
from oracle import seeded_init as si

from conftest import load_golden

needs_ref = pytest.mark.skipif(not shim.available(), reason="reference tree not present")


def rnd(seed, *shape):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def checksum(sd):
    return float(sum(v.double().abs().sum() for v in sd.values()))


def msnet3d(seed=1):
    cfg = shim.load_cfg("cfgs/msnet/msnet3d_sceneflow.yaml").MODEL
    m = oms.load_reference("stereo.modeling.models.msnet.MSNet3D").MSNet3D(cfg).eval()
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=seed, scale=oms.MSNET3D_SCALE))
    return m


# ------------------------------------------------------------------------------------------ oracle vs fixtures
def test_oracle_block_golden():
    g = load_golden("msnet_block")
    for i, (cin, chid, cout, stride) in enumerate(((40, 120, 32, 1), (32, 64, 64, 2))):
        m = oms.MobileV2Residual3D(cin, cout, stride, chid / cin).eval()
        m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=g["seed%d" % i]))
        with torch.no_grad():
            assert torch.equal(m(g["x%d" % i]), g["out%d" % i])


def test_oracle_aggregation_golden():
    g = load_golden("msnet_aggregation")
    m = oms.Aggregation().eval()
    sd = si.seeded_state_dict(m.state_dict(), seed=g["weight_seed"], scale=oms.MSNET3D_SCALE)
    assert checksum(sd) == pytest.approx(g["checksum"], rel=1e-12)
    m.load_state_dict(sd)
    with torch.no_grad():
        assert torch.equal(m.logits(g["volume"]), g["logits"])
        assert torch.equal(m(g["volume"], 32, 32), g["disp"])


def test_oracle_use_res_connect_is_false_for_int_strides():
    """The reference compares its int stride with (1, 1, 1): no block MSNet3D builds adds its identity."""
    m = oms.Aggregation()
    blocks = [b for b in m.modules() if isinstance(b, oms.MobileV2Residual3D)]
    assert len(blocks) == 22 and not any(b.use_res_connect for b in blocks)


# ------------------------------------------------------------------------------------------ oracle vs live reference
@needs_ref
def test_reference_blocks_never_add_identity():
    blocks = [b for b in msnet3d().modules() if type(b).__name__ == "MobileV2_Residual_3D"]
    assert len(blocks) == 22 and not any(b.use_res_connect for b in blocks)


@needs_ref
@pytest.mark.parametrize("cfg", [(40, 120, 32, 1), (32, 64, 64, 2), (128, 256, 128, 1)])
@pytest.mark.parametrize("res", [False, True])
def test_oracle_pins_block(cfg, res):
    cin, chid, cout, stride = cfg
    rsub = oms.load_reference("stereo.modeling.models.msnet.submodule")
    ref, mine = rsub.MobileV2_Residual_3D(cin, cout, stride, chid / cin).eval(), oms.MobileV2Residual3D(cin, cout, stride, chid / cin).eval()
    sd = si.seeded_state_dict(ref.state_dict(), seed=3)
    ref.load_state_dict(sd), mine.load_state_dict(sd)
    ref.use_res_connect = mine.use_res_connect = res and stride == 1 and cin == cout
    x = rnd(4, 2, cin, 3, 5, 6)
    with torch.no_grad():
        assert torch.equal(ref(x), mine(x))


@needs_ref
def test_oracle_pins_model_golden():
    g = load_golden("msnet3d_model")
    m = msnet3d(g["weight_seed"])
    assert checksum(m.state_dict()) == pytest.approx(g["checksum"], rel=1e-12)
    with torch.no_grad():
        want = m({"left": g["left"], "right": g["right"]})["disp_pred"]
        assert torch.equal(want, g["disp"])
        got = oms.eval_forward(m.feature_extraction, oms.aggregation_of(m), g["left"], g["right"])["disp_pred"]
    assert torch.equal(got, want) and want.std() > 1


# ------------------------------------------------------------------------------------------ C ABI and ops
def test_new_entry_point_bound():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib, ops
    assert "osb_mbv2_block3d_fwd" in _lib.SIGNATURES and hasattr(_lib.lib, "osb_mbv2_block3d_fwd")
    args = [16 * (i + 1) for i in range(12)]                           # distinct, 16-byte aligned, never dereferenced

    def call(ptrs=args, B=1, cin=32, chid=96, cout=32, d=4, h=4, w=4, stride=1, lin=0, lout=0):
        _lib.call("osb_mbv2_block3d_fwd", *ptrs, B, cin, chid, cout, d, h, w, stride, lin, lout, None)
    with pytest.raises(ValueError, match="null pointer"):
        call([None] * 12)
    with pytest.raises(ValueError, match="null pointer"):
        call(args[:7] + [None] + args[8:])
    with pytest.raises(ValueError, match=r"\(32, 96, 32, 2\) is not instantiated"):
        call(stride=2)
    with pytest.raises(ValueError, match=r"\(48, 96, 32, 1\) is not instantiated"):
        call(cin=48)
    with pytest.raises(ValueError, match="stride=3"):
        call(stride=3)
    with pytest.raises(ValueError, match="layouts"):
        call(lout=2)
    with pytest.raises(ValueError, match="empty shape"):
        call(d=0)
    t = lambda *s: torch.randn(*s)                                      # noqa: E731
    wts = (t(32, 96), t(96), t(96), t(27, 96), t(96), t(96), t(96, 32), t(32), t(32))
    with pytest.raises(RuntimeError, match="not implemented on the CPU"):
        ops.mbv2_block3d(t(1, 32, 3, 4, 5), *wts)
    with pytest.raises(RuntimeError, match="no backward"):
        ops.mbv2_block3d(torch.randn(1, 32, 3, 4, 5, requires_grad=True), *wts)


def test_packer_refuses_unsupported_blocks():
    from openstereo_b200.aggregation import MSNet3DAggregation, _MBV2Block3D
    with pytest.raises(NotImplementedError, match="blk.*expanse_ratio == 1"):
        _MBV2Block3D(oms.MobileV2Residual3D(32, 32, 1, 1).eval(), "blk")
    with pytest.raises(NotImplementedError, match=r"blk has \(Cin, Chid, Cout, stride\) = \(32, 96, 64, 1\)"):
        _MBV2Block3D(oms.MobileV2Residual3D(32, 64, 1, 3).eval(), "blk")
    m = oms.MobileV2Residual3D(32, 32, 1, 2).eval()
    m.conv[3] = torch.nn.Conv3d(64, 64, 3, 1, 1, groups=32, bias=False)
    with pytest.raises(NotImplementedError, match="blk is not the block"):
        _MBV2Block3D(m, "blk")
    agg = oms.Aggregation().eval()
    agg.encoder_decoder2.redir2 = oms.MobileV2Residual3D(64, 64, 1, 1)
    with pytest.raises(NotImplementedError, match="encoder_decoder2.redir2"):
        MSNet3DAggregation(agg)


# ------------------------------------------------------------------------------------------ patch() contract
def _inputs(h, w, seed, b=1):
    g = torch.Generator().manual_seed(seed)
    return {"left": torch.randn(b, 3, h, w, generator=g), "right": torch.randn(b, 3, h, w, generator=g)}


@needs_ref
def test_patch_msnet3d_contract():
    from openstereo_b200.patch import patch, _patch_msnet3d, _PATCHERS
    assert _PATCHERS["MSNet3D"] is _patch_msnet3d
    m = msnet3d()
    keys = list(m.state_dict().keys())
    x = _inputs(64, 128, 3)
    with torch.no_grad():
        want = m(dict(x))["disp_pred"]
        assert patch(m, strict=False) is m and m._osb_patched and "forward" in vars(m)
        assert patch(m, strict=False) is m                              # idempotent
        assert list(m.state_dict().keys()) == keys
        assert torch.equal(m(dict(x))["disp_pred"], want)               # CPU call delegated to the reference's own forward
        strict = patch(msnet3d())
        with pytest.raises(RuntimeError, match="CUDA inference only"):
            strict(dict(x))


@needs_ref
def test_patch_msnet3d_refuses_expanse_ratio_1():
    from openstereo_b200.patch import patch
    rsub = oms.load_reference("stereo.modeling.models.msnet.submodule")
    m = msnet3d()
    m.encoder_decoder3.redir1 = rsub.MobileV2_Residual_3D(32, 32, 1, 1)
    with pytest.raises(NotImplementedError, match="encoder_decoder3.redir1 uses the expanse_ratio == 1 branch"):
        patch(m, strict=False)
    assert not getattr(m, "_osb_patched", False) and "forward" not in vars(m)
