"""GPU: CoEx on the sm_90a kernels -- the fused regression tail and the nearest resampling against the CPU oracle
(oracle/coex.py, pinned bit-exactly to the reference), CoExAggregation at three level shapes, and patch() on the unmodified
reference class."""
import pytest
import torch
import torch.nn.functional as F

from oracle import _reference_shim as shim
from oracle import coex as ocx
from oracle import seeded_init as si

from conftest import load_golden

pytestmark = pytest.mark.gpu

EPE_BAR = 1e-3
REG_BAR = 1e-4                  # px, regression tail on the same logits
AGG_BAR = 1e-5                  # max |err| / max |want| of the aggregation logits


@pytest.fixture(scope="module")
def osb():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib, ops
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return _lib, ops


def rnd(seed, *shape):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def distinct_logits(seed, b, d, h, w):
    """Logits without exact ties along D (a permutation of 0.3 * [0, D) plus noise below the 0.3 spacing): at D > 16 the reference's
    CPU sort orders exact ties in an implementation-defined way, so comparisons on the reference's order need tie-free logits."""
    g = torch.Generator().manual_seed(seed)
    return torch.rand(b, 1, d, h, w, generator=g).argsort(2).float() * 0.3 + torch.rand(b, 1, d, h, w, generator=g) * 0.2


def one_hot_centre(b, h, w):
    """Superpixel weights that keep only the centre tap: the output is then 4 * disp_4 of the pixel's own cell."""
    spx = torch.zeros(b, 9, h, w)
    spx[:, 4] = 1.0
    return spx


# ------------------------------------------------------------------------------------------------ regression tail
@pytest.mark.parametrize("k", [2, 3, 8])
@pytest.mark.parametrize("logits", [True, False])
def test_regression_vs_oracle(osb, k, logits):
    _, ops = osb
    b, d, h, w = 2, 48, 19, 37                                          # not multiples of the 16 x 32 CTA tile
    cost = distinct_logits(1, b, d, h, w)
    raw = rnd(2, b, 9, 4 * h, 4 * w) * 2
    prob = torch.softmax(raw, 1)
    want = ocx.regression(cost, prob, k)
    got = ops.coex_regression(cost.cuda(), (raw if logits else prob).cuda(), k, spx_is_logits=logits).cpu()
    err = (got - want).abs().max().item()
    print("coex_regression k=%d logits=%s: max |err| %.2e px" % (k, logits, err))
    assert got.shape == want.shape and err <= REG_BAR


@pytest.mark.parametrize("k", [2, 3])
def test_regression_golden_ties(osb, k):
    """The fixture's small-integer logits tie often.  With the centre tap alone, a different choice among tied values would move
    4 * disp_4 by at least 4 / k px, so agreement within REG_BAR means the kernel chose exactly the reference's indices."""
    _, ops = osb
    g = load_golden("coex_regression")
    got = ops.coex_regression(g["cost"].cuda(), g["spx"].cuda(), k).cpu()
    assert (got - g["out_k%d" % k]).abs().max().item() <= REG_BAR
    b, _, _, h, w = g["cost"].shape
    spx = one_hot_centre(b, 4 * h, 4 * w)
    want = ocx.regression(g["cost"], spx, k)
    got = ops.coex_regression(g["cost"].cuda(), spx.cuda(), k).cpu()
    assert (got - want).abs().max().item() <= REG_BAR


def test_regression_selection_on_random_logits(osb):
    _, ops = osb
    cost = distinct_logits(3, 2, 48, 21, 33)
    spx = one_hot_centre(2, 84, 132)
    for k in (2, 3, 8):
        want = ocx.regression(cost, spx, k)
        got = ops.coex_regression(cost.cuda(), spx.cuda(), k).cpu()
        assert (got - want).abs().max().item() <= REG_BAR


def test_regression_ties_lower_index_first_at_d48(osb):
    """At CoEx's D = 48 exact ties go to the lower index (a stable descending sort), at every k."""
    _, ops = osb
    cost = torch.randint(-2, 2, (2, 1, 48, 9, 11), generator=torch.Generator().manual_seed(5)).float()
    spx = one_hot_centre(2, 36, 44)
    for k in (2, 3, 8):
        want = ocx.regression(cost, spx, k, stable=True)
        got = ops.coex_regression(cost.cuda(), spx.cuda(), k).cpu()
        assert (got - want).abs().max().item() <= REG_BAR


# ------------------------------------------------------------------------------------------------ nearest resampling
@pytest.mark.parametrize("src,size", [((1, 1, 7, 136, 12), (6, 135, 24)), ((2, 3, 13, 14, 26), (12, 13, 25)),
                                      ((1, 2, 24, 24, 48), (48, 48, 48)), ((1, 4, 6, 7, 30), (5, 13, 30)),
                                      ((2, 1, 9, 5, 3), (4, 10, 8))])
def test_nearest_resize3d_bit_equal(osb, src, size):
    _, ops = osb
    x = rnd(4, *src).cuda()
    assert torch.equal(ops.nearest_resize3d(x, size), F.interpolate(x, size=size, mode="nearest"))


def test_nearest_resize3d_golden(osb):
    _, ops = osb
    g = load_golden("coex_nearest")
    for i in range(3):
        size = tuple(int(v) for v in g["size%d" % i])
        assert torch.equal(ops.nearest_resize3d(g["x"].cuda(), size).cpu(), g["out%d" % i])


def test_attention_volume_golden(osb):
    _, ops = osb
    g = load_golden("coex_attention")
    got = ops.coex_attention_volume(g["x"].cuda(), g["y"].cuda(), g["maxdisp"], g["head"]).cpu()
    assert got.shape == g["out"].shape and (got - g["out"]).abs().max().item() <= 1e-6


# ------------------------------------------------------------------------------------------------ aggregation engine
def _ceil(n, k):
    return -(-n // k)


def _agg_inputs(b, h, w, seed):
    img = [rnd(seed, b, 96, h, w), rnd(seed + 1, b, 64, _ceil(h, 2), _ceil(w, 2)), rnd(seed + 2, b, 192, _ceil(h, 4), _ceil(w, 4)),
           rnd(seed + 3, b, 160, _ceil(h, 8), _ceil(w, 8))]
    return img, rnd(seed + 4, b, 1, 48, h, w) * 0.3


def _check_aggregation(osb, b, h, w, gce, seed):
    lib, _ = osb
    from openstereo_b200.aggregation import CoExAggregation
    m = ocx.Aggregation(192, gce=gce).eval()
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=seed))
    img, cost = _agg_inputs(b, h, w, seed + 10)
    with torch.no_grad():
        want = m(img, cost)
        eng = CoExAggregation(m.cuda())
        before = lib.launch_count()
        got = eng([t.cuda() for t in img], cost.cuda()).cpu()
        launches = lib.launch_count() - before
    rel = ((got - want).abs().max() / want.abs().max()).item()
    print("CoExAggregation B=%d %dx%d gce=%s: max rel err %.2e, %d launches" % (b, h, w, gce, rel, launches))
    assert got.shape == want.shape and rel <= AGG_BAR
    return launches


@pytest.mark.parametrize("b,h,w", [(2, 64, 128), (1, 135, 240), (1, 50, 64)])
def test_aggregation_vs_oracle(osb, b, h, w):
    launches = _check_aggregation(osb, b, h, w, True, 50)
    assert launches >= 16                                               # every Conv3d / ConvTranspose3d is a launch of its own


def test_aggregation_without_gates(osb):
    _check_aggregation(osb, 1, 50, 64, False, 51)


# ------------------------------------------------------------------------------------------------ patch() on the reference
needs_ref = pytest.mark.skipif(not shim.available(), reason="reference tree (oracle/_ref) not staged")


def _coex():
    shim.install_timm_stub()
    cfg = shim.load_cfg("cfgs/coex/coex_sceneflow_amp.yaml").MODEL
    m = shim.load("stereo.modeling.models.coex.coex").CoEx(cfg).eval()
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=1))
    return m


def _inputs(b, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return {"left": torch.randn(b, 3, h, w, generator=g), "right": torch.randn(b, 3, h, w, generator=g)}


def patched_vs_reference(lib, b, h, w, seed):
    """-> (EPE px, reference disparity std, launches, selection flips): the reference on the CPU vs patch() on the GPU."""
    from openstereo_b200.patch import patch
    m = _coex()
    seen = []
    m.DispProcessor.register_forward_pre_hook(lambda mod, args: seen.append(args[0]["cost_volume"].detach().cpu()))
    x = _inputs(b, h, w, seed)
    with torch.no_grad():
        want = m(dict(x))["disp_pred"]
        patch(m.cuda())
        before = lib.launch_count()
        got = m({k: v.cuda() for k, v in x.items()})["disp_pred"]
        launches = lib.launch_count() - before
    assert got.shape == want.shape and got.is_cuda
    assert seen[1].shape == seen[0].shape                              # inputs['cost_volume'] keeps the reference's shape
    k = m.DispProcessor.regression.top_k
    sel = [ocx.topk_pool(c, k)[1].sort(2)[0] for c in seen]
    flips = int((sel[0] != sel[1]).any(2).sum())
    epe = (got.cpu() - want).abs().mean().item()
    print("patch(CoEx) B=%d %dx%d: EPE %.3e px vs the reference on the CPU (disp std %.2f), %d launches, %d low-resolution pixels "
          "with a different top-%d selection" % (b, h, w, epe, want.std().item(), launches, flips, k))
    return epe, want.std().item(), launches


@needs_ref
def test_patch_coex_256x512(osb):
    lib, _ = osb
    epe, std, launches = patched_vs_reference(lib, 1, 256, 512, 60)
    assert launches >= 16 + 3 + 1 and std > 1 and epe <= EPE_BAR       # 16 aggregation convs, the volume (2 norms + 1), the tail


@needs_ref
def test_patch_coex_never_reaches_kernels_when_recording_or_training(osb):
    """strict=False: a CUDA call that autograd records, or a training call, runs the reference's own code (no launch of this
    library) with gradients intact; strict=True refuses both loudly."""
    lib, _ = osb
    from openstereo_b200.patch import patch
    x = {k: v.cuda() for k, v in _inputs(2, 128, 256, 61).items()}
    m = patch(_coex().cuda(), strict=False)
    before = lib.launch_count()
    out = m(dict(x))["disp_pred"]
    assert lib.launch_count() == before and out.requires_grad
    out.mean().backward()
    assert any(p.grad is not None and p.grad.abs().sum() > 0 for n, p in m.named_parameters() if n.startswith("Backbone."))
    m.train()
    before = lib.launch_count()
    out = m(dict(x))
    assert lib.launch_count() == before
    out["disp_pred"].mean().backward()
    strict = patch(_coex().cuda())
    with pytest.raises(RuntimeError, match="CUDA inference only"):
        strict(dict(x))
    with pytest.raises(RuntimeError, match="CUDA inference only"):
        strict.train()(dict(x))
