"""Stage the UNMODIFIED reference under ``oracle/_ref/`` (git-ignored; never part of the repository).

The reference (AntreasAntoniou/HowToTrainYourMAMLPytorch) is a pure-Python program without packaging metadata
(no setup.py / pyproject.toml), so ``pip install --target oracle/_ref <reference checkout>`` has nothing to build; what an
install would amount to is making its modules importable from one directory, which is what this script does: it copies
the reference's own ``.py`` modules (and its ``utils`` package) byte for byte.  Nothing is edited, nothing of it is
committed -- ``oracle/_ref/`` is in ``.gitignore`` -- and ``MANIFEST.json`` records the sha256 of every staged file.

  python oracle/stage_reference.py [REFERENCE_DIR]

Without REFERENCE_DIR the first of $MAML_REFERENCE_DIR, a ``reference`` checkout next to this repository and
``/root/reference`` (where the project's build environment keeps the reference checkout) that exists is used; without
any of them nothing is staged and ``stage()`` returns None (``__graft_entry__.build()`` then warns on stderr).  ``bench.py --impl reference``, the ``cpu_baseline`` / ``torch_gpu_baseline`` legs (through
``baseline/run_reference.py``) and the ExperimentBuilder test import the staged copy, and skip or fall back without it.
"""
import hashlib
import json
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
DEST = os.path.join(HERE, "_ref")
CANDIDATES = [c for c in (os.environ.get("MAML_REFERENCE_DIR"), os.path.join(os.path.dirname(HERE), "..", "reference"),
                            "/root/reference") if c]
DEFAULT_SRC = next((c for c in CANDIDATES if os.path.isdir(c)), CANDIDATES[0])
MODULES = ["few_shot_learning_system.py", "meta_neural_network_architectures.py", "inner_loop_optimizers.py",
           "experiment_builder.py", "data.py", "train_maml_system.py",
           os.path.join("utils", "__init__.py"), os.path.join("utils", "parser_utils.py"),
           os.path.join("utils", "storage.py"), os.path.join("utils", "dataset_tools.py")]


def stage(src=DEFAULT_SRC):
    src = os.path.abspath(src)
    if not os.path.isdir(src):
        return None
    manifest = {}
    for rel in MODULES:
        s, d = os.path.join(src, rel), os.path.join(DEST, rel)
        os.makedirs(os.path.dirname(d), exist_ok=True)
        shutil.copyfile(s, d)
        with open(d, "rb") as fh:
            manifest[rel] = hashlib.sha256(fh.read()).hexdigest()
    cfg_src, cfg_dst = os.path.join(src, "experiment_config"), os.path.join(DEST, "experiment_config")
    if os.path.isdir(cfg_src):
        shutil.copytree(cfg_src, cfg_dst, dirs_exist_ok=True)
    sub = os.path.join(src, ".SUBMODULES.json")
    commit = None
    if os.path.exists(sub):
        try:
            commit = json.load(open(sub)).get("commit")
        except Exception:
            commit = None
    with open(os.path.join(DEST, "MANIFEST.json"), "w") as fh:
        json.dump({"source": src, "commit": commit, "sha256": manifest}, fh, indent=1)
    return DEST


if __name__ == "__main__":
    out = stage(sys.argv[1] if len(sys.argv) > 1 else DEFAULT_SRC)
    print(out if out else "reference sources not found; nothing staged")
