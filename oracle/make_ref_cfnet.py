"""Recipe: stage the UNMODIFIED reference files of CFNet (cfnet/cfnet.py, cfnet/submodule.py) under oracle/_ref/, next to what
oracle/make_ref.py stages, so that the CFNet tests and tools/bench_configs.py c17 can build the reference's own classes from
the unchanged YAML where the reference tree is absent.

    python oracle/make_ref_cfnet.py      (needs the reference tree; run after oracle/make_ref.py, which prunes
                                          oracle/_ref/ down to its own manifest)

Byte copies; CFNET_MANIFEST.json lists their sha256 sums.  TEST / MEASUREMENT INFRASTRUCTURE ONLY.
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

DIRS = ["stereo/modeling/models/cfnet"]
FILES = ["cfgs/cfnet/cfnet_sceneflow_part2.yaml"]


def _sha(path):
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


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
    with open(os.path.join(DEST, "CFNET_MANIFEST.json"), "w") as f:
        json.dump({"source": SRC, "files": manifest}, f, indent=1, sort_keys=True)
    if verbose:
        print("oracle/_ref: %d CFNet files" % len(manifest))
    return DEST


if __name__ == "__main__":
    make(verbose=True)
    sys.exit(0)
