"""CPU: the C-ABI shared library loads, exports every symbol include/openstereo_b200.h declares, and the
host-side argument checks behave like the reference's (no compute without a GPU)."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def native():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib
    return _lib


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "openstereo_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(osb_[a-z0-9_]+)\s*\(", text)))


def test_header_symbols_exported(native):
    names = declared_symbols()
    assert len(names) >= 13
    lib = ctypes.CDLL(native.LIB_PATH)
    for name in names:
        assert hasattr(lib, name), "%s declared in the header but not exported" % name
    # every compute entry point bound by the Python layer is declared in the header
    for name in native.SIGNATURES:
        assert name in names


def test_binding_signatures_match_header(native):
    """Arity and C types of every ctypes binding are checked against the prototypes in the header."""
    text = open(os.path.join(ROOT, "include", "openstereo_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    kinds = {"const float*": ctypes.c_void_p, "float*": ctypes.c_void_p, "const void*": ctypes.c_void_p, "int": ctypes.c_int, "float": ctypes.c_float,
             "osb_stream_t": ctypes.c_void_p, "long long": ctypes.c_longlong}
    for name, argtypes in native.SIGNATURES.items():
        m = re.search(r"int\s+%s\s*\(([^)]*)\)" % name, text)
        assert m, name
        params = [p.strip() for p in m.group(1).replace("\n", " ").split(",")]
        want = []
        for p in params:
            ctype = p.rsplit(" ", 1)[0].strip()
            assert ctype in kinds, (name, p)
            want.append(kinds[ctype])
        assert want == list(argtypes), "%s: header %d params vs binding %d" % (name, len(want), len(argtypes))


def test_version_and_error_channel(native):
    assert native.lib.osb_abi_version() == 1
    assert native.launch_count() >= 0
    # argument validation happens before any CUDA call: a null pointer is OSB_EINVAL -> ValueError
    with pytest.raises(ValueError, match="null pointer"):
        native.call("osb_gwc_volume_fwd", None, None, None, 1, 8, 4, 4, 4, 2, None)


def test_persistent_grid_cap_and_variant_hooks(native):
    """Test hooks of the persistent kernels: declared in the header, bound with their C types, host-only state (no device needed)."""
    from openstereo_b200 import ops
    names = declared_symbols()
    assert "osb_set_persistent_grid_cap" in names and "osb_tc_last_variant" in names and "osb_volume_last_variant" in names
    assert native.lib.osb_set_persistent_grid_cap.argtypes == [ctypes.c_int]
    assert native.lib.osb_set_persistent_grid_cap.restype is ctypes.c_int
    assert native.lib.osb_tc_last_variant.restype is ctypes.c_char_p
    assert native.lib.osb_volume_last_variant.restype is ctypes.c_char_p
    assert ops.set_persistent_grid_cap(3) == 0
    assert ops.set_persistent_grid_cap(-2) == 3                  # negative = no cap
    assert ops.set_persistent_grid_cap(0) == 0
    assert isinstance(ops.tc_last_variant(), str)
    assert isinstance(ops.volume_last_variant(), str)


def test_ops_refuse_cpu_tensors(native):
    from openstereo_b200 import ops
    x = torch.randn(1, 8, 4, 16)
    with pytest.raises(RuntimeError, match="not implemented on the CPU"):
        ops.build_gwc_volume(x, x, 4, 2)
    with pytest.raises(RuntimeError, match="not implemented on the CPU"):
        ops.softargmin(torch.randn(1, 4, 4, 4), 4)
    with pytest.raises(ValueError, match="expected 4D input"):
        ops.faster_soft_argmin(torch.randn(4, 4, 4), 4)          # psmnet_disp_processor.py:56-58
    with pytest.raises(NotImplementedError):
        ops.cat_fms(x, x, max_disp=4, start_disp=-1)


_A = 0x10000                                     # a 16-byte aligned address; no call below gets past the argument check
TC_FWD_CALLS = {                                  # every tensor-core entry point on a shape it serves, x misaligned by 4 bytes
    "conv3d": ("osb_conv3d_k3_tc_fwd", lambda x: (x, _A, _A, None, None, _A, 1, 32, 32, 2, 4, 128, 0, 1, 1, None)),
    "conv3d-kc16": ("osb_conv3d_k3_tc_fwd", lambda x: (x, _A, _A, None, None, _A, 1, 32, 64, 2, 4, 64, 0, 1, 1, None)),
    "conv3d-gate": ("osb_conv3d_k3_tc_gate_fwd", lambda x: (x, _A, _A, None, None, _A, _A, 1, 32, 64, 2, 4, 64, 0, None)),
    "conv3d-slice": ("osb_conv3d_k3_tc_cs_fwd", lambda x: (x, _A, _A, None, None, None, _A, 1, 32, 96, 2, 4, 16, 0, 160, None)),
    "conv3d-ncdhw": ("osb_conv3d_k3_tc_ncdhw_fwd", lambda x: (x, _A, _A, None, None, _A, 1, 32, 32, 2, 4, 128, 0, 1, 1, None)),
    "conv2d": ("osb_conv2d_k3_tc_fwd", lambda x: (x, _A, _A, None, None, _A, 1, 32, 64, 4, 128, 1, 0, 1, 1, None)),
    "conv2d-dil2": ("osb_conv2d_k3_tc_fwd", lambda x: (x, _A, _A, None, None, _A, 1, 32, 128, 4, 128, 2, 0, 1, 1, None)),
    "conv3d-s2": ("osb_conv3d_k3_s2_tc_fwd", lambda x: (x, _A, _A, None, None, _A, 1, 32, 64, 2, 4, 128, 0, 1, 1, None)),
    "conv3d-s2-slice": ("osb_conv3d_k3_s2_tc_cs_fwd", lambda x: (x, _A, _A, None, _A, 1, 32, 96, 2, 4, 32, 0, 160, None)),
    "deconv3d-k3": ("osb_deconv3d_k3_tc_fwd", lambda x: (x, _A, _A, None, None, _A, 1, 64, 32, 2, 4, 64, 0, 1, 1, None)),
    "deconv3d-k4": ("osb_deconv3d_k4_tc_fwd", lambda x: (x, _A, _A, None, None, _A, 1, 64, 32, 32, 2, 4, 64, 0, 1, 1, None)),
    "deconv3d-k4-slice": ("osb_deconv3d_k4_tc_cs_fwd", lambda x: (x, _A, _A, None, _A, 1, 32, 64, 2, 4, 16, 0, 96, None)),
}


@pytest.mark.skipif(torch.cuda.is_available(), reason="a missing check would launch a kernel on a fake address")
@pytest.mark.parametrize("case", sorted(TC_FWD_CALLS))
def test_tc_entry_points_refuse_misaligned_pointers(native, case):
    """The tensor-core kernels load and store 16 bytes at a time and bulk-copy rows: every entry point refuses a misaligned operand
    as an argument error, before any CUDA call."""
    name, args = TC_FWD_CALLS[case]
    with pytest.raises(ValueError, match="16-byte aligned"):
        native.call(name, *args(_A + 4))


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "openstereo_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f
