"""TEST INFRASTRUCTURE ONLY: builds oracle/liboracle_port.so and, when the reference is present,
oracle/_ref/liboracle_ref.so (see oracle/Makefile) and the staged copy oracle/_ref/reference (stage_reference); the
restatements of the point-cloud utilities (port_lib) and their reference-side libraries (ref_lib)."""
import ctypes as C
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
PORT_SO = os.path.join(HERE, "liboracle_port.so")
REF_SO = os.path.join(HERE, "_ref", "liboracle_ref.so")
# the parts of the reference that the C++ layer and the GPU-side test binaries compile against, staged by
# stage_reference() so that they travel with oracle/_ref to a machine without the reference tree
STAGED_REF = os.path.join(HERE, "_ref", "reference")
STAGED_PARTS = (("3rdparty", "Eigen"), ("demos",), ("tests", "externalAppTest"))
_SOURCE_ROOT = os.environ.get("S4_REFERENCE_ROOT", "/root/reference")
REFERENCE_ROOT = _SOURCE_ROOT if os.path.isdir(_SOURCE_ROOT) or not os.path.isdir(STAGED_REF) else STAGED_REF


def stage_reference():
    """Copies STAGED_PARTS of the reference (Eigen, the host-side dependency of the C++ API; the demo mains, the PCL
    wrapper and the MeshLab plugin; the packaging test's main) into oracle/_ref/reference when the reference is present
    and they are not staged yet.  Returns the root the C++ layer and the test binaries are to be built against: the
    reference itself, else the staged copy, else None."""
    if os.path.isdir(os.path.join(_SOURCE_ROOT, "3rdparty", "Eigen", "Eigen")) and \
            os.path.realpath(_SOURCE_ROOT) != os.path.realpath(STAGED_REF):
        for part in STAGED_PARTS:
            dst = os.path.join(STAGED_REF, *part)
            if not os.path.isdir(dst):
                tmp = dst + ".tmp"
                shutil.rmtree(tmp, ignore_errors=True)
                shutil.copytree(os.path.join(_SOURCE_ROOT, *part), tmp, copy_function=shutil.copyfile)
                for dp, dns, _ in os.walk(tmp):
                    os.chmod(dp, 0o755)
                os.rename(tmp, dst)
        return _SOURCE_ROOT
    if os.path.isdir(os.path.join(STAGED_REF, "3rdparty", "Eigen", "Eigen")):
        return STAGED_REF
    return None


def _stale(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.exists(s) and os.path.getmtime(s) > t for s in sources)


def _env():
    """the environment of every compiler call here: g++ itself, whatever CXX and CC name"""
    env = dict(os.environ)
    env.pop("CXX", None)
    env.pop("CC", None)
    return env


_libs = {}


def _lib(path):
    if path not in _libs:
        _libs[path] = C.CDLL(path)
    return _libs[path]


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def eigen_root():
    """the Eigen that code compiled against include/super4pcs/ needs: S4_EIGEN_ROOT, the reference's copy or the
    system's; None when there is none"""
    for c in (os.environ.get("S4_EIGEN_ROOT"), os.path.join(REFERENCE_ROOT, "3rdparty", "Eigen"),
              "/usr/include/eigen3"):
        if c and os.path.exists(os.path.join(c, "Eigen", "Core")):
            return c
    return None


_PORT_FLAGS = ("-std=c++11", "-O2", "-ffp-contract=off", "-fopenmp")
# the restatements of the point-cloud utilities: name -> (compile flags, the ports besides oracle/<name>_port.cc that
# its library holds).  tests/build_shim.py compiles each oracle/<name>_port.cc into the CPU stand-in with these flags.
PORTS = {
    "nearest": (_PORT_FLAGS, ()),
    "nearest_any": (_PORT_FLAGS, ()),
    "range": (_PORT_FLAGS, ()),
    "knn": (_PORT_FLAGS, ()),
    "normals": (_PORT_FLAGS, ("knn",)),
    "orient_normals": (_PORT_FLAGS, ("knn",)),
    "outliers": (_PORT_FLAGS, ("knn",)),
    "clusters": (_PORT_FLAGS, ()),
    # -O3: the CPU baseline of scripts/planes_bench.py
    "planes": (("-std=c++11", "-O3", "-ffp-contract=off", "-fopenmp"), ()),
    # one thread, although the source has an OpenMP pragma: the CPU baseline of scripts/voxel_grid_bench.py
    "voxel_grid": (("-std=c++11", "-O2", "-ffp-contract=off"), ()),
    "fpfh": (("-std=c++17", "-O2", "-ffp-contract=off", "-fopenmp"), ("knn",)),  # C++17 for its hex-float literals
}


def port_src(name):
    return os.path.join(HERE, name + "_port.cc")


def port_lib(name, force=False):
    """oracle/liboracle_<name>.so, the restatement PORTS[name], rebuilt when it is older than its sources"""
    flags, others = PORTS[name]
    srcs = [port_src(n) for n in (name,) + others]
    so = os.path.join(HERE, "liboracle_%s.so" % name)
    if force or _stale(so, srcs):
        subprocess.check_call(["g++", *flags, "-fPIC", "-shared", *srcs, "-o", so], env=_env())
    return so


# the queries whose reference side is the reference's own kd-tree, in oracle/<name>_ref.cc
REF_LIBS = ("nearest", "nearest_any", "range")


def ref_lib(name, force=False):
    """oracle/_ref/liboracle_ref_<name>.so (oracle/<name>_ref.cc linked against build_ref()'s library), or None when it
    can be neither built (no reference sources) nor found"""
    src = os.path.join(HERE, name + "_ref.cc")
    so = os.path.join(HERE, "_ref", "liboracle_ref_%s.so" % name)
    ref = REFERENCE_ROOT
    base = build_ref()
    if base is not None and os.path.isdir(os.path.join(ref, "src", "super4pcs")) and (force or _stale(so, [src, base])):
        # the flags of oracle/Makefile's reference build (the reference's Release configuration)
        subprocess.check_call(["g++", "-std=c++11", "-O3", "-DNDEBUG", "-fopenmp", "-DSUPER4PCS_USE_OPENMP",
                               "-DEIGEN_DONT_PARALLELIZE", "-I", os.path.join(ref, "src"),
                               "-I", os.path.join(ref, "3rdparty", "Eigen"), "-fPIC", "-w", "-shared", src,
                               "-o", so, "-L", os.path.dirname(base), "-loracle_ref", "-Wl,-rpath,$ORIGIN"], env=_env())
    return so if os.path.exists(so) else None


def build_port(force=False):
    if force or _stale(PORT_SO, [os.path.join(HERE, "port.cc")]):
        subprocess.check_call(["make", "-C", HERE, "port"], stdout=subprocess.DEVNULL)
    return PORT_SO


def build_ref(force=False):
    """Returns the path of the reference oracle, or None when it cannot be built here
    (no /root/reference on the GPU box) and no prebuilt copy travelled with the repo."""
    have_ref = os.path.isdir(os.path.join(REFERENCE_ROOT, "src", "super4pcs"))
    if have_ref and (force or _stale(REF_SO, [os.path.join(HERE, "ref_harness.cc")])):
        subprocess.check_call(["make", "-C", HERE, "ref", "REF=" + REFERENCE_ROOT],
                              stdout=subprocess.DEVNULL)
    return REF_SO if os.path.exists(REF_SO) else None


DROPIN_SO = os.path.join(HERE, "_dropin", "libb200_harness.so")


def build_dropin_harness(force=False):
    """The SAME harness source (oracle/ref_harness.cc, written against the reference's headers)
    compiled unchanged against the PRODUCT's header-compatible layer (include/super4pcs/ +
    libsuper4pcs_b200.so): the drop-in proof tests/test_dropin_gpu.py drives.  Test infrastructure:
    the dependency points from here to the product, never the other way.  Needs Eigen (host-side API
    dependency); without it the prebuilt copy that travelled with the repo is used."""
    root = os.path.dirname(HERE)
    libdir = os.path.join(root, "super4pcs_b200", "lib")
    prod = os.path.join(libdir, "libsuper4pcs_b200.so")
    eig = eigen_root()
    src = os.path.join(HERE, "ref_harness.cc")
    if eig and os.path.exists(prod) and (force or _stale(DROPIN_SO, [src, prod])):
        os.makedirs(os.path.dirname(DROPIN_SO), exist_ok=True)
        subprocess.check_call(["g++", "-std=c++14", "-O3", "-DNDEBUG", "-fPIC", "-w", "-fopenmp", "-DSUPER4PCS_USE_OPENMP",
                               "-shared", "-I", os.path.join(root, "include"), "-I", eig, src, "-o", DROPIN_SO,
                               "-L", libdir, "-lsuper4pcs_b200", "-ls4g", "-Wl,-rpath,$ORIGIN/../../super4pcs_b200/lib"], env=_env())
    return DROPIN_SO if os.path.exists(DROPIN_SO) else None
