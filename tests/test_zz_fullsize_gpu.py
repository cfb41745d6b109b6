"""GPU, last in collection order: end-to-end parity of the host mirrors at the BENCH configurations (256x512, D = 192), where
every tensor-core route is live at once, against the CPU oracle with the same seeded weights.  Bar: the north star's 1e-3 px EPE.

The tensor core's fp32 accumulation truncates, so every conv comes out slightly too small, and the shrink adds up coherently over
the ~80 layers in front of a sharp 192-bin softmax.  The unbiased operand split + the expected-loss correction of the epilogues
(csrc/tc_common.cuh) keep it inside the bar."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import models as omodels       # noqa: E402
from oracle import seeded_init as si       # noqa: E402

EPE_BAR = 1e-3
GWC_CFG = {"MAX_DISP": 192, "USE_CONCAT_VOLUME": True, "CONCAT_CHANNELS": 12, "DOWNSAMPLE": 4, "NUM_GROUPS": 40}


@pytest.fixture(scope="module")
def osb():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib, host_models
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return _lib, host_models


def _pairs(b, seed):
    g = torch.Generator().manual_seed(seed)
    return {"left": torch.randn(b, 3, 256, 512, generator=g), "right": torch.randn(b, 3, 256, 512, generator=g)}


def _gwc_models(hm):
    oracle = omodels.GwcNet(192, True, 12, 4, 40).eval()
    sd = si.seeded_state_dict(oracle.state_dict(), seed=1, scale=si.GWCNET_SCALE)
    oracle.load_state_dict(sd)
    mine = hm.GwcNet(GWC_CFG).eval()
    mine.load_state_dict(sd)
    return oracle, mine.cuda()


@pytest.mark.parametrize("tc_backbone", [True, False])
def test_gwcnet_bench_configuration_epe(osb, tc_backbone):
    """BASELINE config 2, one pair.  tc_backbone=True: the 2D extractor's residual blocks on the wgmma kernels as well (86
    launches); False: the extractor on cuDNN, the in-scope hot path (volume, aggregation, tail) on this library (33 launches)."""
    lib, hm = osb
    oracle, mine = _gwc_models(hm)
    x = _pairs(1, 0)
    old = hm.USE_TC_BACKBONE
    hm.USE_TC_BACKBONE = tc_backbone
    try:
        with torch.no_grad():
            want = oracle(dict(x))["disp_pred"]
            before = lib.launch_count()
            got = mine({k: v.cuda() for k, v in x.items()})["disp_pred"]
            launches = lib.launch_count() - before
    finally:
        hm.USE_TC_BACKBONE = old
    assert got.shape == want.shape == (1, 256, 512)
    e = (got.cpu() - want).abs().mean().item()
    print("GwcNet 256x512 (backbone on %s) EPE vs oracle: %.3e px, %d launches of this library" % (
        "wgmma" if tc_backbone else "cuDNN", e, launches))
    assert launches >= (80 if tc_backbone else 30)
    assert want.std() > 10 and e <= EPE_BAR


def test_gwcnet_bench_batch8_epe(osb):
    """The batch the bench times: B = 8 distinct pairs in one forward (per-image EPE, every image under the bar)."""
    _, hm = osb
    oracle, mine = _gwc_models(hm)
    x = _pairs(8, 123)
    with torch.no_grad():
        want = torch.cat([oracle({k: v[i:i + 1] for k, v in x.items()})["disp_pred"] for i in range(8)])
        got = mine({k: v.cuda() for k, v in x.items()})["disp_pred"].cpu()
    per_image = (got - want).abs().mean(dim=(1, 2))
    print("GwcNet B=8 256x512 per-image EPE vs oracle: max %.3e mean %.3e px" % (per_image.max().item(), per_image.mean().item()))
    assert want.std() > 10 and per_image.max().item() <= EPE_BAR


def test_psmnet_config1_epe(osb):
    """BASELINE config 1: PSMNet, one pair at 256x512 (W' = 128: the wgmma stem / backbone routes that 256x256 never took)."""
    lib, hm = osb
    oracle = omodels.PSMNet(192).eval()
    sd = si.seeded_state_dict(oracle.state_dict(), seed=1, scale=si.PSMNET_SCALE, keep=si.PSMNET_KEEP)
    oracle.load_state_dict(sd)
    mine = hm.PSMNet({"MAX_DISP": 192}).eval()
    mine.load_state_dict(sd)
    mine.cuda()
    x = _pairs(1, 7)
    with torch.no_grad():
        want = oracle(dict(x))
        before = lib.launch_count()
        got = mine({k: v.cuda() for k, v in x.items()})
        launches = lib.launch_count() - before
    errs = [(g.cpu() - w).abs().mean().item() for g, w in zip(got["train_preds"], want["train_preds"])]
    print("PSMNet 256x512 EPE vs oracle (disp1, disp2, disp3): %s px, %d launches" % (", ".join("%.3e" % e for e in errs), launches))
    assert want["disp_pred"].std() > 10 and max(errs) <= EPE_BAR
