"""Recipe: stage the unchanged MSNet2D YAML of the reference under oracle/_ref/, next to the msnet package that
oracle/make_ref_msnet.py stages, so that the MSNet2D tests and tools/bench_configs.py c18 can build the reference's own class where
the reference tree is absent.

    python oracle/make_ref_msnet2d.py      (needs the reference tree; run after oracle/make_ref.py, which prunes oracle/_ref/)

Byte copies; MSNET2D_MANIFEST.json lists their sha256 sums.  TEST / MEASUREMENT INFRASTRUCTURE ONLY.
"""
import hashlib
import json
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
DEST = os.path.join(HERE, "_ref")
SRC = os.environ.get("OPENSTEREO_REFERENCE_SRC", "/root/reference")

FILES = ["cfgs/msnet/msnet2d_sceneflow.yaml", "stereo/modeling/models/msnet/MSNet2D.py", "stereo/modeling/models/msnet/submodule.py"]


def _sha(path):
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


def make(verbose=False):
    if not os.path.isdir(os.path.join(SRC, "stereo", "modeling")):
        raise RuntimeError("reference tree not found at %s" % SRC)
    manifest = {}
    for rel in FILES:
        src = os.path.join(SRC, rel)
        if not os.path.exists(src):
            raise RuntimeError("missing reference file %s" % rel)
        dst = os.path.join(DEST, rel)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        if not (os.path.exists(dst) and _sha(dst) == _sha(src)):
            shutil.copyfile(src, dst)
        manifest[rel] = _sha(dst)
    with open(os.path.join(DEST, "MSNET2D_MANIFEST.json"), "w") as f:
        json.dump({"source": SRC, "files": manifest}, f, indent=1, sort_keys=True)
    if verbose:
        print("oracle/_ref: %d MSNet2D files" % len(manifest))
    return DEST


if __name__ == "__main__":
    make(verbose=True)
    sys.exit(0)
