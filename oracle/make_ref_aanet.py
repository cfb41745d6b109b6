"""Recipe: stage the UNMODIFIED reference files of AANet (the model package, the DCNv2 extension's Python wrapper and CUDA sources,
and both YAMLs) under oracle/_ref/, and compile the extension (deform_conv_cuda) for sm_90a next to its wrapper, so that the
AANet tests and tools/bench_configs.py c16 can run the reference's own model -- and its own deformable-convolution kernel -- where
the reference tree is absent.

    python oracle/make_ref_aanet.py     (needs the reference tree; run after oracle/make_ref.py, which prunes oracle/_ref/ down
                                         to its own manifest)

Byte copies; AANET_MANIFEST.json lists their sha256 sums.  make_ref.py's prune removes the compiled module with every other file
it does not list, so the build lives in a per-user cache directory keyed by the sha256 of the two sources and the torch version:
the two-minute compile runs once per source change, and every later call copies the cached module back.  TEST / MEASUREMENT
INFRASTRUCTURE ONLY.
"""
import glob
import hashlib
import json
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
DEST = os.path.join(HERE, "_ref")
SRC = os.environ.get("OPENSTEREO_REFERENCE_SRC", "/root/reference")

DIRS = ["stereo/modeling/models/aanet", "stereo/libs/AANet/deform_conv"]
FILES = ["cfgs/aanet/aanet_sceneflow.yaml", "cfgs/aanet/aanet_sceneflow_uniform.yaml",
         "stereo/libs/AANet/deform_conv/src/deform_conv_cuda.cpp", "stereo/libs/AANet/deform_conv/src/deform_conv_cuda_kernel.cu"]
EXT_DIR = "stereo/libs/AANet/deform_conv"
EXT_SOURCES = ["src/deform_conv_cuda.cpp", "src/deform_conv_cuda_kernel.cu"]
EXT_NAME = "deform_conv_cuda"


def _sha(path):
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


def extension_path(root=DEST):
    """Where the compiled reference extension sits: next to the staged deform_conv.py that imports it."""
    return os.path.join(root, EXT_DIR, EXT_NAME + ".so")


def _compile(sources, verbose):
    import torch
    from torch.utils import cpp_extension
    key = hashlib.sha256(("".join(_sha(s) for s in sources) + torch.__version__).encode()).hexdigest()[:16]
    cache = os.path.join(os.environ.get("XDG_CACHE_HOME") or os.path.join(os.path.expanduser("~"), ".cache"),
                         "openstereo_b200", "aanet_ext", key)
    built = os.path.join(cache, EXT_NAME + ".so")
    if not os.path.exists(built):
        os.makedirs(cache, exist_ok=True)
        saved = os.environ.get("TORCH_CUDA_ARCH_LIST")
        os.environ["TORCH_CUDA_ARCH_LIST"] = "9.0a"                # -gencode arch=compute_90a,code=sm_90a only
        try:
            cpp_extension.load(EXT_NAME, sources, build_directory=cache, verbose=verbose, is_python_module=False)
        finally:
            if saved is None:
                os.environ.pop("TORCH_CUDA_ARCH_LIST")
            else:
                os.environ["TORCH_CUDA_ARCH_LIST"] = saved
    return built


def make(verbose=False):
    if not os.path.isdir(os.path.join(SRC, "stereo", "modeling")):
        raise RuntimeError("reference tree not found at %s" % SRC)
    wanted = list(FILES)
    for d in DIRS:
        wanted += sorted(os.path.relpath(p, SRC) for p in glob.glob(os.path.join(SRC, d, "*.py")))
    manifest = {}
    for rel in wanted:
        src = os.path.join(SRC, rel)
        if not os.path.exists(src):
            raise RuntimeError("missing reference file %s" % rel)
        dst = os.path.join(DEST, rel)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        if not (os.path.exists(dst) and _sha(dst) == _sha(src)):
            shutil.copyfile(src, dst)
        manifest[rel] = _sha(dst)
    built = _compile([os.path.join(DEST, EXT_DIR, s) for s in EXT_SOURCES], verbose)
    shutil.copyfile(built, extension_path())
    with open(os.path.join(DEST, "AANET_MANIFEST.json"), "w") as f:
        json.dump({"source": SRC, "files": manifest, "extension": _sha(extension_path())}, f, indent=1, sort_keys=True)
    if verbose:
        print("oracle/_ref: %d AANet files and %s" % (len(manifest), os.path.relpath(extension_path(), DEST)))
    return DEST


if __name__ == "__main__":
    make(verbose=True)
    sys.exit(0)
