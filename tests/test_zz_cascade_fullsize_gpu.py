"""GPU, full size: one CasPSMNet pair at the cfg's eval crop 512x960 (cfgs/casnet/casnet_psm_sceneflow.yaml unchanged,
seeded weights) through patch(), against the reference on the CPU.  Bar: the north star's 1e-3 px EPE."""
import pytest
import torch

from oracle import _reference_shim as shim
from oracle import cascade as ocas
from oracle import seeded_init as si

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not shim.available(), reason="reference tree (oracle/_ref) not staged")]


def test_patch_casnet_512x960():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib
    from openstereo_b200.patch import patch
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    cfg = shim.load_cfg("cfgs/casnet/casnet_psm_sceneflow.yaml").MODEL
    m = shim.load("stereo.modeling.models.casnet.cas_psm").PSMNet(cfg).eval()
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=1, scale=ocas.CASNET_SCALE))
    g = torch.Generator().manual_seed(50)
    x = {"left": torch.randn(1, 3, 512, 960, generator=g), "right": torch.randn(1, 3, 512, 960, generator=g)}
    with torch.no_grad():
        want = m(dict(x))["disp_pred"]
        patch(m.cuda())
        before = _lib.launch_count()
        got = m({k: v.cuda() for k, v in x.items()})["disp_pred"]
        launches = _lib.launch_count() - before
    e = (got.cpu() - want).abs().mean().item()
    print("patch(CasPSMNet) 512x960 EPE vs the reference on CPU: %.3e px (disp std %.2f), %d launches" % (e, want.std().item(), launches))
    assert launches >= 2 * (1 + 20 + 1) and want.std() > 1 and e <= 1e-3
