"""Recipe: compile the REFERENCE's own Cython MISE (code/src/libmise/mise.pyx — the only native source in the reference,
SURVEY §2.2) from a checkout of the reference named by $HOLD_REFERENCE into oracle/_ref/ (git-ignored, never copied into the
repo's history).  Used only to pin the MISE restatement (tests/test_cpu_mise.py); nothing at build, test or bench run time
needs the reference.  usage: python oracle/build_ref_mise.py"""
import os
import subprocess
import sys
import sysconfig

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(os.environ.get("HOLD_REFERENCE", ""), "code/src/libmise/mise.pyx")
OUT = os.path.join(HERE, "_ref")


def build():
    if not os.environ.get("HOLD_REFERENCE") or not os.path.exists(SRC):
        return None
    os.makedirs(OUT, exist_ok=True)
    ext = sysconfig.get_config_var("EXT_SUFFIX")
    so = os.path.join(OUT, "mise" + ext)
    if os.path.exists(so) and os.path.getmtime(so) >= os.path.getmtime(SRC):
        return so
    cpp = os.path.join(OUT, "mise.cpp")
    subprocess.run([sys.executable, "-m", "cython", "--cplus", "-3", SRC, "-o", cpp], check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    import numpy as np

    inc = [sysconfig.get_paths()["include"], np.get_include()]
    cmd = ["g++", "-O2", "-shared", "-fPIC", "-std=c++14", "-w"] + [f"-I{i}" for i in inc] + ["-o", so, cpp]
    subprocess.run(cmd, check=True)
    os.remove(cpp)
    return so


if __name__ == "__main__":
    print(build())
