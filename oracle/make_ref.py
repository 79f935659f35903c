"""TEST INFRASTRUCTURE - recipe that materialises the UNMODIFIED reference under oracle/_ref/.

    python -m oracle.make_ref            (needs the reference checkout; run by __graft_entry__.build())

The reference is six pure-Python files with no package metadata (no setup.py / pyproject, so the
`pip install` has nothing to install) and nothing to compile.
This recipe copies `learner.py models.py utils.py actor.py train.py` byte for byte from where
they lie in the reference checkout ($IMPALA_REFERENCE_DIR) into `oracle/_ref/` - a build OUTPUT directory: git-ignored (no
reference source ever enters the history), shipped with the built .so to
wherever the GPU tests run - and writes the two stub modules the reference imports but this image lacks
(`gym` -> the in-repo old-API CartPole of oracle/cartpole_env.py, `pybullet_envs` -> empty).

With oracle/_ref/ present, `bench.py --impl reference` and the `cpu_baseline` leg time the real
`learner.Learner._learn` (`cpu_baseline.kind = "reference"`), and `tests/test_gpu_reference_train.py`
runs the reference's own train.py / actor.py against the GPU learner.
"""
from __future__ import annotations

import hashlib
import json
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF_OUT = os.path.join(HERE, "_ref")
SRC = os.environ.get("IMPALA_REFERENCE_DIR", "/root/reference")
FILES = ("learner.py", "models.py", "utils.py", "actor.py", "train.py")

GYM_STUB = '''"""Stub written by oracle/make_ref.py: the image has no gym.  `make` returns the in-repo CartPole
with the OLD gym API the reference expects (utils.py:95-107, actor.py:73,88)."""
from oracle.cartpole_env import CartPoleEnv as Env  # noqa: F401  (utils.py:112 annotation)
from oracle.cartpole_env import make  # noqa: F401
'''


def make(verbose: bool = True) -> str | None:
    if not os.path.isfile(os.path.join(SRC, "learner.py")):
        if verbose:
            print(f"[make_ref] {SRC} not present: keeping whatever is in {REF_OUT}")
        return REF_OUT if os.path.isfile(os.path.join(REF_OUT, "learner.py")) else None
    os.makedirs(os.path.join(REF_OUT, "gym"), exist_ok=True)
    os.makedirs(os.path.join(REF_OUT, "pybullet_envs"), exist_ok=True)
    manifest = {}
    for f in FILES:
        shutil.copyfile(os.path.join(SRC, f), os.path.join(REF_OUT, f))
        with open(os.path.join(REF_OUT, f), "rb") as fh:
            manifest[f] = hashlib.sha256(fh.read()).hexdigest()
    with open(os.path.join(REF_OUT, "gym", "__init__.py"), "w") as fh:
        fh.write(GYM_STUB)
    with open(os.path.join(REF_OUT, "pybullet_envs", "__init__.py"), "w") as fh:
        fh.write('"""Empty stub written by oracle/make_ref.py (utils.py:7 imports it for its side effects)."""\n')
    with open(os.path.join(REF_OUT, "MANIFEST.json"), "w") as fh:
        json.dump(dict(source=SRC, sha256=manifest), fh, indent=1)
    if verbose:
        print(f"[make_ref] copied {len(FILES)} files from {SRC} -> {REF_OUT}")
    return REF_OUT


if __name__ == "__main__":
    sys.exit(0 if make() else 1)
