"""Recipe: stage the UNMODIFIED reference files of every model the tests and benchmarks build from the reference's own classes
under oracle/_ref/, so they travel to the GPU box, and compile AANet's DCNv2 extension (deform_conv_cuda) for sm_90a next to its
wrapper.

    python oracle/make_ref.py            (needs the reference tree at $OPENSTEREO_REFERENCE_SRC, default /root/reference)

oracle/_ref/ is git-ignored (never committed -- the repository holds no reference source) but ships with the working tree,
exactly like the in-tree .so.  Files are byte copies, copied only when their sha256 differs; MANIFEST.json lists every staged file's sha256 (and the extension's), and every other file under oracle/_ref/ is
deleted, so a stale copy cannot survive.  Importing this module does not import torch; only the extension compile does.
TEST / MEASUREMENT INFRASTRUCTURE ONLY: nothing under openstereo_b200/ reads oracle/_ref.
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

# per model, relative to the reference root: "dirs" stage their *.py, "trees" every *.py below them, "files" one file each
MODELS = {
    # GwcNet / PSMNet / StereoBase / LightStereo / IGEV: tests/test_patch_gpu.py and the other tests of these models,
    # bench.py --impl reference, its cpu_baseline and its GPU comparators (fast_foundationstereo's Triton gwc kernel)
    "core": {"dirs": ["stereo/modeling/cost_volume", "stereo/modeling/disp_pred", "stereo/modeling/common",
                      "stereo/modeling/disp_refinement", "stereo/modeling/backbones", "stereo/modeling/models/gwcnet",
                      "stereo/modeling/models/psmnet", "stereo/modeling/models/stereobase", "stereo/modeling/models/igev",
                      "stereo/modeling/models/lightstereo"],
             "files": ["stereo/modeling/models/fast_foundationstereo/core/submodule.py",
                       "stereo/modeling/models/igevpp/submodule.py", "stereo/modeling/models/casnet/submodule.py",
                       "stereo/evaluation/metric_per_image.py", "tools/measure.py",
                       "cfgs/gwcnet/gwcnet_sceneflow.yaml", "cfgs/psmnet/psmnet_sceneflow.yaml",
                       "cfgs/stereobase/stereobase_sceneflow.yaml", "cfgs/lightstereo/lightstereo_s_sceneflow.yaml",
                       "cfgs/igev/igev_sceneflow_amp.yaml"]},
    # CasPSMNet / CasGwcNet: the cascade tests, tools/bench_configs.py c6
    "cascade": {"dirs": ["stereo/modeling/models/casnet"], "files": ["cfgs/casnet/casnet_psm_sceneflow.yaml"]},
    # the CoEx tests, bench_configs c7
    "coex": {"dirs": ["stereo/modeling/models/coex"], "files": ["cfgs/coex/coex_sceneflow_amp.yaml"]},
    # the MSNet3D tests, bench_configs c8
    "msnet3d": {"dirs": ["stereo/modeling/models/msnet"], "files": ["cfgs/msnet/msnet3d_sceneflow.yaml"]},
    # the MSNet2D tests, bench_configs c18
    "msnet2d": {"files": ["cfgs/msnet/msnet2d_sceneflow.yaml", "stereo/modeling/models/msnet/MSNet2D.py",
                          "stereo/modeling/models/msnet/submodule.py"]},
    # the IGEV-RT tests, bench_configs c9
    "igev_rt": {"dirs": ["stereo/modeling/models/igev_rt"],
                "files": ["cfgs/igev_rt/igev_rt_sceneflow_uniform.yaml", "cfgs/igev_rt/igev_rt_sceneflow_amp.yaml"]},
    # the IGEV++ tests, bench_configs c12
    "igevpp": {"dirs": ["stereo/modeling/models/igevpp"],
               "files": ["cfgs/igevpp/igevpp_sceneflow_uniform.yaml", "cfgs/igevpp/igevpp_sceneflow_amp.yaml"]},
    # the MonSter tests, bench_configs c13; the model imports its depth_anything_v2/ tree
    "monster": {"trees": ["stereo/modeling/models/monster"],
                "files": ["cfgs/monster/monster_sceneflow_uniform.yaml", "cfgs/monster/monster_sceneflow.yaml"]},
    # the AANet tests, bench_configs c16: the model, the DCNv2 wrapper and the sources of its extension (EXT_* below)
    "aanet": {"dirs": ["stereo/modeling/models/aanet", "stereo/libs/AANet/deform_conv"],
              "files": ["cfgs/aanet/aanet_sceneflow.yaml", "cfgs/aanet/aanet_sceneflow_uniform.yaml",
                        "stereo/libs/AANet/deform_conv/src/deform_conv_cuda.cpp",
                        "stereo/libs/AANet/deform_conv/src/deform_conv_cuda_kernel.cu"]},
    # the CFNet tests, bench_configs c17
    "cfnet": {"dirs": ["stereo/modeling/models/cfnet"], "files": ["cfgs/cfnet/cfnet_sceneflow_part2.yaml"]},
}
EXT_DIR = "stereo/libs/AANet/deform_conv"
EXT_SOURCES = ["src/deform_conv_cuda.cpp", "src/deform_conv_cuda_kernel.cu"]
EXT_NAME = "deform_conv_cuda"


def _sha(path):
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


def reference_present():
    return os.path.isdir(os.path.join(SRC, "stereo", "modeling"))


def extension_path():
    """Where the compiled reference extension sits: next to the staged deform_conv.py that imports it."""
    return os.path.join(DEST, EXT_DIR, EXT_NAME + ".so")


def _compile(sources, verbose):
    """Build the extension once per source change and torch version, in a per-user cache directory keyed by both."""
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


def _stage(src, rel):
    dst = os.path.join(DEST, rel)
    os.makedirs(os.path.dirname(dst), exist_ok=True)
    if not (os.path.exists(dst) and _sha(dst) == _sha(src)):
        shutil.copyfile(src, dst)
    return _sha(dst)


def make(verbose=False):
    if not reference_present():
        raise RuntimeError("reference tree not found at %s" % SRC)
    wanted = set()
    for entry in MODELS.values():
        wanted.update(entry.get("files", ()))
        for d in entry.get("dirs", ()):
            wanted.update(os.path.relpath(p, SRC) for p in glob.glob(os.path.join(SRC, d, "*.py")))
        for d in entry.get("trees", ()):
            wanted.update(os.path.relpath(p, SRC) for p in glob.glob(os.path.join(SRC, d, "**", "*.py"), recursive=True))
    manifest = {}
    for rel in sorted(wanted):
        if not os.path.exists(os.path.join(SRC, rel)):
            raise RuntimeError("missing reference file %s" % rel)
        manifest[rel] = _stage(os.path.join(SRC, rel), rel)
    ext = os.path.relpath(extension_path(), DEST)
    ext_sha = _stage(_compile([os.path.join(DEST, EXT_DIR, s) for s in EXT_SOURCES], verbose), ext)
    keep = set(manifest) | {ext, "MANIFEST.json"}
    for r, _, fs in os.walk(DEST):
        for f in fs:
            if os.path.relpath(os.path.join(r, f), DEST) not in keep:
                os.remove(os.path.join(r, f))
    head = ""
    try:
        with open(os.path.join(SRC, ".git", "HEAD")) as f:
            head = f.read().strip()
    except OSError:
        pass
    with open(os.path.join(DEST, "MANIFEST.json"), "w") as f:
        json.dump({"source": SRC, "git_head": head, "files": manifest, "extension": ext_sha}, f, indent=1, sort_keys=True)
    if verbose:
        size = sum(os.path.getsize(os.path.join(DEST, r)) for r in manifest)
        print("oracle/_ref: %d files (%d bytes) and %s" % (len(manifest), size, ext))
    return DEST


if __name__ == "__main__":
    make(verbose=True)
    sys.exit(0)
