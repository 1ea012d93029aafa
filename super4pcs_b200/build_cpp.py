"""Builds the header-compatible C++ layer (include/super4pcs/, cpp/) on top of libs4g.so:

  super4pcs_b200/lib/libsuper4pcs_b200.so   Match4PCSBase / MatchSuper4PCS / IOManager
  super4pcs_b200/lib/externalAppTest        the reference's packaging test (tests/externalAppTest/main.cpp), unchanged
  super4pcs_b200/lib/Super4PCS              the REFERENCE's own demo main, compiled unchanged from
                                            /root/reference/demos/Super4PCS/super4pcs_test.cc
                                            against OUR headers (only where /root/reference exists)

(The TestMatcher-style probe used by tests/test_dropin_gpu.py is test infrastructure and is built by
the test side, not here.)

Eigen (a host-side dependency of the public API types, e.g. Eigen::Ref<Matrix4f>) is taken from
S4_EIGEN_ROOT or the vendored copy of the reference named by S4_REFERENCE_ROOT (the driver's build() points it at a
staged copy where the reference tree is absent); without any, binaries built earlier are used as they are.
"""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIBDIR = os.path.join(HERE, "lib")
REFERENCE_ROOT = os.environ.get("S4_REFERENCE_ROOT", "/root/reference")
CXX = "g++"
FLAGS = ["-std=c++14", "-O3", "-DNDEBUG", "-fPIC", "-w"]


def eigen_root():
    for c in (os.environ.get("S4_EIGEN_ROOT"), os.path.join(REFERENCE_ROOT, "3rdparty", "Eigen"), "/usr/include/eigen3"):
        if c and os.path.exists(os.path.join(c, "Eigen", "Core")):
            return c
    return None


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


def _headers():
    out = []
    for dp, _, fns in os.walk(os.path.join(ROOT, "include")):
        out += [os.path.join(dp, f) for f in fns]
    return out


def _run(cmd):
    env = dict(os.environ)
    env.pop("CXX", None)
    env.pop("CC", None)
    r = subprocess.run(cmd, env=env, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("build failed:\n%s\n%s" % (" ".join(cmd), r.stderr[-4000:]))


def build_all(force=False):
    eig = eigen_root()
    lib = os.path.join(LIBDIR, "libsuper4pcs_b200.so")
    demo = os.path.join(LIBDIR, "Super4PCS")
    if eig is None:
        ext = os.path.join(LIBDIR, "externalAppTest")
        return {"lib": lib if os.path.exists(lib) else None, "demo": demo if os.path.exists(demo) else None,
                "external_app_test": ext if os.path.exists(ext) else None}
    inc = ["-I", os.path.join(ROOT, "include"), "-I", eig]
    srcs = [os.path.join(ROOT, "cpp", f) for f in ("match4pcsBase.cc", "super4pcs.cc", "pair_order.cc", "io.cc",
                                                      "normals.cc", "outliers.cc", "clusters.cc",
                                                      "planes.cc", "voxel_grid.cc", "orient_normals.cc",
                                                      "features.cc")]
    link = ["-L", LIBDIR, "-ls4g", "-pthread", "-Wl,-rpath,$ORIGIN"]
    private = [os.path.join(ROOT, "cpp", f) for f in os.listdir(os.path.join(ROOT, "cpp")) if f.endswith(".h")]
    if force or _stale(lib, srcs + private + _headers() + [os.path.join(LIBDIR, "libs4g.so")]):
        _run([CXX, *FLAGS, "-shared", *inc, *srcs, "-o", lib, *link])
    link2 = ["-L", LIBDIR, "-lsuper4pcs_b200", "-ls4g", "-Wl,-rpath,$ORIGIN"]
    ref_demo = os.path.join(REFERENCE_ROOT, "demos", "Super4PCS", "super4pcs_test.cc")
    if os.path.exists(ref_demo) and (force or _stale(demo, [lib, ref_demo])):
        _run([CXX, *FLAGS, *inc, "-I", os.path.join(REFERENCE_ROOT, "demos"), ref_demo, "-o", demo, *link2])
    # the reference's packaging test (tests/externalAppTest/main.cpp), also compiled unchanged
    ext = os.path.join(LIBDIR, "externalAppTest")
    ref_ext = os.path.join(REFERENCE_ROOT, "tests", "externalAppTest", "main.cpp")
    if os.path.exists(ref_ext) and (force or _stale(ext, [lib, ref_ext])):
        _run([CXX, *FLAGS, *inc, ref_ext, "-o", ext, *link2])
    return {"lib": lib, "demo": demo if os.path.exists(demo) else None,
            "external_app_test": ext if os.path.exists(ext) else None}


if __name__ == "__main__":
    print(build_all(force=True))
