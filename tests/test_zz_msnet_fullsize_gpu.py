"""GPU, full size: patch(MSNet3D) at the cfg's 512x960 eval crop against the unpatched reference on the CPU (slow: the CPU
reference runs every MobileV2_Residual_3D block unfused)."""
import pytest
import torch

from oracle import _reference_shim as shim

from test_msnet_gpu import EPE_BAR, patched_vs_reference

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not shim.available(), reason="reference tree (oracle/_ref) not staged")]


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib
    torch.backends.cudnn.allow_tf32 = False
    return _lib


def test_patch_msnet3d_512x960(lib):
    epe, std = patched_vs_reference(lib, 1, 512, 960, 40)
    assert std > 1 and epe <= EPE_BAR
