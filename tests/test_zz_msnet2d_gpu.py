"""GPU: MSNet2D on the library (aggregation.MSNet2DVolume / MSNet2DAggregation) and the interlaced-crop mode of the volume kernel.

* osb_interlaced_crops_fwd is a row family of tests/test_kernel_contract_gpu.py ("crop": bit-exact against the fp64 gather of
  oracle/msnet2d.py in a NaN-guarded buffer, both staging instantiations, grid caps, the other item order, the refusals); here the
  existing volume entry points with the mode off still give exact copies / the oracle's correlations.
* The volume front end against the reference's own 48-iteration loop in fp64: per voxel the error stays below 1e-4 times the
  largest voxel plus 1e-5, and every voxel with w < d is exactly 0.  Crops below OSB_TC_MIN_WIDTH take the CUDA-core kernels.
* The aggregation stage and the whole patched model against the unpatched model (cuDNN fp32, TF32 off): EPE <= 1e-3 px at
  256 x 512 and 512 x 960; the fp16-range guard of the front end's tensor-core layers.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def osb():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib, aggregation, ops
    return _lib, aggregation, ops


@pytest.fixture(autouse=True)
def _fp32_reference():
    cudnn, matmul = torch.backends.cudnn, torch.backends.cuda.matmul
    old = cudnn.allow_tf32, matmul.allow_tf32, cudnn.deterministic, cudnn.benchmark
    cudnn.allow_tf32 = matmul.allow_tf32 = False
    cudnn.deterministic, cudnn.benchmark = True, False
    yield
    cudnn.allow_tf32, matmul.allow_tf32, cudnn.deterministic, cudnn.benchmark = old


def _feats(b, c, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(b, c, h, w, generator=g), torch.randn(b, c, h, w, generator=g)


def test_existing_volumes_unchanged(osb):
    _, _, ops = osb
    from oracle import cost_volume as ocv
    fl, fr = _feats(2, 12, 5, 70, seed=3)
    for mask in (True, False):
        got = ops.build_concat_volume(fl.cuda(), fr.cuda(), 24, mask_left=mask).cpu()
        b, c, h, w = fl.shape
        want = torch.zeros(b, 2 * c, 24, h, w)
        for d in range(24):
            want[:, :c, d, :, d:] = fl[..., d:]
            if not mask:
                want[:, :c, d, :, :d] = fl[..., :d]
            want[:, c:, d, :, d:] = fr[..., :w - d]
        assert torch.equal(got, want)
    g1, g2 = _feats(1, 40, 4, 64, seed=4)
    got = ops.build_gwc_volume(g1.cuda(), g2.cuda(), 20, 10).cpu()
    assert (got - ocv.build_gwc_volume(g1, g2, 20, 10)).abs().max().item() <= 1e-6


def _model():
    from oracle.msnet2d import reference_model
    return reference_model()


@pytest.mark.parametrize("hw", [(16, 128), (8, 56), (32, 240)])
def test_front_end_against_the_reference_loop(osb, hw):
    """(8, 56): crops 56 .. 9 columns wide, those below 24 on the CUDA-core kernels; (16, 128): the W = 128 routes."""
    _, aggregation, _ = osb
    from oracle.msnet2d import volume_loop
    h, w = hw
    m = _model()
    fl, fr = _feats(2, 32, h, w, seed=h + w)
    fl, fr = fl * 0.3, fr * 0.3                                          # the scale of preconv11's outputs
    with torch.no_grad():
        want = volume_loop(m.double(), fl.double(), fr.double())
        m.float().cuda()
        eng = aggregation.MSNet2DVolume(m)
        got = eng(fl.cuda(), fr.cuda()).cpu().double()
    assert got.shape == want.shape and float(want.std()) > 0.05
    tri = torch.ones(48, w).triu() == 0
    assert torch.all(got.permute(0, 2, 1, 3)[:, :, tri] == 0), "the left triangle is not exactly zero"
    err = (got - want).abs().max().item()
    assert err <= 1e-4 * want.abs().max().item() + 1e-5, err
    narrow = [d for d in range(48) if not eng.tc_width(w - d)]
    assert (w < 72) == bool(narrow)


def _pair(b, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return {"left": torch.randn(b, 3, h, w, generator=g).cuda(), "right": torch.randn(b, 3, h, w, generator=g).cuda()}


def test_aggregation_stage(osb):
    _, aggregation, _ = osb
    m = _model().cuda()
    data = _pair(2, 128, 256, seed=7)
    with torch.no_grad():
        fl = m.preconv11(m.feature_extraction(data["left"]))
        fr = m.preconv11(m.feature_extraction(data["right"]))
        from oracle.msnet2d import volume_loop
        volume = volume_loop(m, fl, fr)
        cost0 = m.dres0(volume)
        cost0 = m.dres1(cost0) + cost0
        want = m.classif3(m.encoder_decoder3(m.encoder_decoder2(m.encoder_decoder1(cost0))))
        eng = aggregation.MSNet2DAggregation(m)
        got = eng.logits(volume)
    assert float(want.std()) > 1.0
    assert (got - want).abs().max().item() <= 1e-4 * want.abs().max().item()


@pytest.mark.parametrize("b,h,w", [(2, 256, 512), (1, 512, 960)])
def test_whole_model(osb, b, h, w):
    from openstereo_b200.patch import patch
    data = _pair(b, h, w, seed=h)
    unpatched, patched = _model().cuda(), patch(_model().cuda())
    with torch.no_grad():
        want = unpatched(data)["disp_pred"]
        got = patched(data)["disp_pred"]
    assert got.shape == want.shape == (b, h, w) and got.dtype == want.dtype
    assert float(want.std()) > 2.0
    epe = (got - want).abs().mean().item()
    assert epe <= 1e-3, epe


def test_range_guard(osb):
    _, aggregation, ops = osb
    m = _model().cuda()
    eng = aggregation.MSNet2DVolume(m)
    fl, fr = (t.cuda() for t in _feats(1, 32, 4, 64, seed=9))
    with torch.no_grad():
        eng(fl, fr)
        torch.cuda.synchronize()
        eng(fl * 1e4, fr * 1e4)                                          # staged operands beyond the +-4094 fp16 range
        torch.cuda.synchronize()
        with pytest.raises(RuntimeError, match="fp16 range"):
            eng(fl, fr)
    assert ops.tc_overflow_count(reset=True) == 0                       # the report reset the counter
