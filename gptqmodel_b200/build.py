"""Build libb2q.so in-tree for sm_90a (`python gptqmodel_b200/build.py`, or `__graft_entry__.build()`)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")


def build(verbose: bool = False, force: bool = False) -> str:
    if force:
        subprocess.run(["make", "-C", CSRC, "clean"], check=True, capture_output=not verbose)
    r = subprocess.run(["make", "-C", CSRC, "-j4"], capture_output=True, text=True)
    if verbose or r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
    if r.returncode != 0:
        raise RuntimeError("building libb2q.so failed")
    out = os.path.join(HERE, "libb2q.so")
    assert os.path.exists(out)
    return out


if __name__ == "__main__":
    print(build(verbose=True, force="--force" in sys.argv))
