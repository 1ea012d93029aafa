"""TEST INFRASTRUCTURE ONLY: builds oracle/liboracle_port.so and, when the reference is present,
oracle/_ref/liboracle_ref.so (see oracle/Makefile) and the staged copy oracle/_ref/reference (stage_reference)."""
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
    eig = None
    for c in (os.environ.get("S4_EIGEN_ROOT"), os.path.join(REFERENCE_ROOT, "3rdparty", "Eigen"), "/usr/include/eigen3"):
        if c and os.path.exists(os.path.join(c, "Eigen", "Core")):
            eig = c
            break
    src = os.path.join(HERE, "ref_harness.cc")
    if eig and os.path.exists(prod) and (force or _stale(DROPIN_SO, [src, prod])):
        os.makedirs(os.path.dirname(DROPIN_SO), exist_ok=True)
        env = dict(os.environ)
        env.pop("CXX", None)
        env.pop("CC", None)
        subprocess.check_call(["g++", "-std=c++14", "-O3", "-DNDEBUG", "-fPIC", "-w", "-fopenmp", "-DSUPER4PCS_USE_OPENMP",
                               "-shared", "-I", os.path.join(root, "include"), "-I", eig, src, "-o", DROPIN_SO,
                               "-L", libdir, "-lsuper4pcs_b200", "-ls4g", "-Wl,-rpath,$ORIGIN/../../super4pcs_b200/lib"], env=env)
    return DROPIN_SO if os.path.exists(DROPIN_SO) else None
