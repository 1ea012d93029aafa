"""TEST INFRASTRUCTURE ONLY: builds tests/_build/libs4g_oracle_shim.so (tests/stubs/s4g_oracle_shim.cc), a
stand-in for libs4g.so answered by the CPU oracle, used through LD_PRELOAD by the CPU tests of the C++ layer to run its
host logic without a GPU.  The restatements of the point-cloud utilities (oracle/<name>_port.cc) are compiled into it,
each with the flags of its oracle library.  Never part of the product."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(HERE, "_build", "libs4g_oracle_shim.so")


def build(force=False):
    from oracle import _build
    port = _build.build_port()
    src = os.path.join(HERE, "stubs", "s4g_oracle_shim.cc")
    ports = {name: _build.port_src(name) for name in _build.PORTS}
    deps = [src, port, os.path.join(ROOT, "include", "s4g.h"), *ports.values()]
    if force or _build._stale(OUT, deps):
        os.makedirs(os.path.dirname(OUT), exist_ok=True)
        objs = []
        for name, cc in ports.items():
            objs.append(os.path.join(os.path.dirname(OUT), name + "_port.o"))
            subprocess.check_call(["g++", *_build.PORTS[name][0], "-fPIC", "-c", cc, "-o", objs[-1]], env=_build._env())
        subprocess.check_call(["g++", "-std=c++14", "-O2", "-ffp-contract=off", "-fopenmp", "-fPIC", "-shared",
                               "-I", os.path.join(ROOT, "include"), src, *objs, "-o", OUT,
                               "-L", os.path.dirname(port), "-loracle_port", "-Wl,-rpath," + os.path.dirname(port)],
                              env=_build._env())
    return OUT


if __name__ == "__main__":
    import sys
    sys.path.insert(0, ROOT)
    print(build(force=True))
