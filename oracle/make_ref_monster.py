"""Recipe: stage the UNMODIFIED reference files of MonSter (the model package with its depth_anything_v2/ tree, and both YAMLs)
under oracle/_ref/, next to what oracle/make_ref.py and the other make_ref_* recipes stage, so that the MonSter tests and
tools/bench_configs.py c13 can build the reference's own class from the unchanged YAMLs where the reference tree is absent.

    python oracle/make_ref_monster.py     (needs the reference tree; run after oracle/make_ref.py, which prunes
                                            oracle/_ref/ down to its own manifest)

Byte copies; MONSTER_MANIFEST.json lists their sha256 sums.  TEST / MEASUREMENT INFRASTRUCTURE ONLY.
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

DIRS = ["stereo/modeling/models/monster"]
FILES = ["cfgs/monster/monster_sceneflow_uniform.yaml", "cfgs/monster/monster_sceneflow.yaml"]


def _sha(path):
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


def make(verbose=False):
    if not os.path.isdir(os.path.join(SRC, "stereo", "modeling")):
        raise RuntimeError("reference tree not found at %s" % SRC)
    wanted = list(FILES)
    for d in DIRS:
        wanted += sorted(os.path.relpath(p, SRC) for p in glob.glob(os.path.join(SRC, d, "**", "*.py"), recursive=True))
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
    with open(os.path.join(DEST, "MONSTER_MANIFEST.json"), "w") as f:
        json.dump({"source": SRC, "files": manifest}, f, indent=1, sort_keys=True)
    if verbose:
        print("oracle/_ref: %d MonSter files" % len(manifest))
    return DEST


if __name__ == "__main__":
    make(verbose=True)
    sys.exit(0)
