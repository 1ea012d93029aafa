"""Builds and runs the test programs tests/cpp/<name>.cc of the C++ layer's utilities.  Each reads its input from a file,
calls the layer and writes what it returned to another file.  The CPU tests run them with the oracle stand-in of libs4g
(tests/build_shim.py) preloaded, the GPU tests on the real library."""
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build(name, outdir):
    """compiles tests/cpp/<name>.cc into `outdir` against the C++ layer; None when the layer or Eigen is missing"""
    from oracle import _build
    from super4pcs_b200 import build_cpp
    if build_cpp.build_all()["lib"] is None:
        return None
    eig = _build.eigen_root()
    if eig is None:
        return None
    libdir = os.path.join(ROOT, "super4pcs_b200", "lib")
    exe = os.path.join(str(outdir), name)
    subprocess.check_call(["g++", "-std=c++14", "-O2", "-w", "-I", os.path.join(ROOT, "include"), "-I", eig,
                           os.path.join(ROOT, "tests", "cpp", name + ".cc"), "-o", exe, "-L", libdir,
                           "-lsuper4pcs_b200", "-ls4g", "-Wl,-rpath," + libdir], env=_build._env())
    return exe


def run(exe, workdir, payload, args, preload=None):
    """runs `exe IN OUT *args` with IN holding the bytes `payload` and LD_PRELOAD=preload -> the bytes of OUT"""
    src, dst = os.path.join(str(workdir), "in.bin"), os.path.join(str(workdir), "out.bin")
    with open(src, "wb") as f:
        f.write(payload)
    env = dict(os.environ)
    if preload:
        env["LD_PRELOAD"] = preload
    r = subprocess.run([exe, src, dst, *args], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.returncode, r.stdout[-2000:], r.stderr[-2000:])
    with open(dst, "rb") as f:
        return f.read()


class Reader:
    """the arrays of a program's output, read one after another"""

    def __init__(self, b):
        self.b, self.at = b, 0

    def take(self, dt, n):
        a = np.frombuffer(self.b, dt, n, self.at).copy()
        self.at += a.nbytes
        return a

    def done(self):
        return self.at == len(self.b)
