"""Builds super4pcs_b200/lib/libs4g.so (hand-written sm_90a CUDA + the extern "C" ABI of
include/s4g.h) IN-TREE with nvcc.  Cross-compiles without a GPU."""
import concurrent.futures as cf
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "lib", "obj")
LIB = os.path.join(HERE, "lib", "libs4g.so")
SOURCES = ["context.cu", "verify.cu", "rigid.cu", "pairs.cu", "quads.cu", "sampler.cu", "comm.cu", "normals.cu", "outliers.cu",
           "query.cu", "clusters.cu", "planes.cu", "voxel_grid.cu", "orient_normals.cu",
           "fpfh.cu"]

NVCC_FLAGS = [
    "-std=c++17", "-O3",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo",
    "-fmad=false",            # parity: the reference binary has no FMA contraction (SURVEY B.1/B.3)
    "-Xcompiler", "-fPIC",
    "-I", os.path.join(ROOT, "include"),
    "-I", CSRC,
]


def _defines():
    """extra -D flags for A/B builds of the kernels (scripts/verify_ab.sh).  The flags of the last build are kept in a
    stamp file next to the objects: a build with other flags (e.g. a default build after a variant) recompiles everything."""
    return os.environ.get("S4G_NVCC_DEFINES", "").split()


def _nvcc():
    for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build_lib(force=False, verbose=False, extra_flags=(), out_dir=None):
    """out_dir: build the objects and the library there instead of in the tree (variant builds that must not replace the
    tree's library, scripts/verify_phases.py); returns the library's path"""
    nvcc = _nvcc()
    obj_dir = OBJ if out_dir is None else os.path.join(out_dir, "obj")
    lib = LIB if out_dir is None else os.path.join(out_dir, "libs4g.so")
    os.makedirs(obj_dir, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(ROOT, "include", "s4g.h"))
    srcs = [s for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    stamp, defines = os.path.join(obj_dir, "defines.txt"), " ".join(_defines())
    if (open(stamp).read() if os.path.exists(stamp) else "") != defines:
        force = True
    extra_flags = tuple(extra_flags) + tuple(_defines())
    if not force and not _stale(lib, [os.path.join(CSRC, s) for s in srcs] + headers):
        return lib                            # prebuilt library is current (e.g. on the GPU box)
    env = dict(os.environ)
    env.pop("CXX", None)
    env.pop("CC", None)
    jobs = []
    for s in srcs:
        src = os.path.join(CSRC, s)
        obj = os.path.join(obj_dir, s.replace(".cu", ".o"))
        if force or _stale(obj, [src] + headers):
            jobs.append([nvcc, *NVCC_FLAGS, *extra_flags, "-c", src, "-o", obj])

    def run(cmd):
        if verbose:
            print(" ".join(cmd), file=sys.stderr)
        r = subprocess.run(cmd, env=env, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed:\n%s\n%s\n%s" % (" ".join(cmd), r.stdout, r.stderr))
        return r.stderr

    with cf.ThreadPoolExecutor(max_workers=max(1, min(len(jobs), os.cpu_count() or 1))) as ex:
        outs = list(ex.map(run, jobs))
    objs = [os.path.join(obj_dir, s.replace(".cu", ".o")) for s in srcs]
    if jobs or force or _stale(lib, objs):
        run([nvcc, "-shared", "-o", lib, *objs, "-gencode", "arch=compute_90a,code=sm_90a",
             "-Xcompiler", "-fPIC", "-cudart", "static"])
    with open(stamp, "w") as f:
        f.write(defines)
    if verbose:
        for o in outs:
            if o:
                print(o, file=sys.stderr)
    return lib


if __name__ == "__main__":
    print(build_lib(force="--force" in sys.argv, verbose=True,
                    extra_flags=("-Xptxas", "-v") if "--ptxas" in sys.argv else ()))
