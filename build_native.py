"""Build the native library in-tree: fast_gicp_b200/lib/libvgicp_b200.so (sm_90a only, -lineinfo).

    python build_native.py [--force] [-v]

Lives outside the package on purpose: importing fast_gicp_b200 requires the built library (no CPU fallback), so the
builder must be importable without it.
"""
import os
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
HERE = os.path.join(ROOT, "fast_gicp_b200")
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libvgicp_b200.so")

GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]  # H100 (Hopper); the image carries no other architecture and no PTX
NVCC_FLAGS = GENCODE + [
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC,-fvisibility=hidden,-O3",
]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


# (source, extra nvcc flags).  vgicp_stage1.cu must not contract a*b+c: its results are compared bit-for-bit.
UNITS = [("vgicp_b200.cu", []), ("vgicp_stage1.cu", ["--fmad=false"])]


def _deps():
    out = [os.path.join(ROOT, "include", "vgicp_b200.h")]
    for f in os.listdir(CSRC):
        if f.endswith((".cu", ".cuh", ".hpp", ".h")):
            out.append(os.path.join(CSRC, f))
    return out


def needs_build():
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    return any(os.path.getmtime(d) > t for d in _deps())


def build_native(force=False, verbose=False):
    if not force and not needs_build():
        return LIB_PATH
    os.makedirs(LIB_DIR, exist_ok=True)
    env = {k: v for k, v in os.environ.items() if k not in ("CC", "CXX")}  # the image's CC wrapper lacks libgomp specs
    ccbin = ["-ccbin", "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"]
    obj_dir = os.path.join(LIB_DIR, "obj")
    os.makedirs(obj_dir, exist_ok=True)
    objs = []
    for src, extra in UNITS:
        obj = os.path.join(obj_dir, src.replace(".cu", ".o"))
        cmd = [_nvcc()] + NVCC_FLAGS + extra + (["-Xptxas", "-v"] if verbose else []) + ccbin + ["-c", "-o", obj, os.path.join(CSRC, src)]
        subprocess.check_call(cmd, env=env)
        objs.append(obj)
    subprocess.check_call([_nvcc()] + GENCODE + ["-shared", "-o", LIB_PATH] + ccbin + objs, env=env)
    return LIB_PATH


PREP_SRC = os.path.join(CSRC, "prep", "vgicp_prep.cu")
PREP_LIB_PATH = os.path.join(LIB_DIR, "libvgicp_prep_b200.so")


def build_prep(force=False):
    """Input-preparation library (include/vgicp_prep_b200.h): lib/libvgicp_prep_b200.so, independent of libvgicp_b200.so."""
    hdr = os.path.join(ROOT, "include", "vgicp_prep_b200.h")
    if not force and os.path.exists(PREP_LIB_PATH) and all(os.path.getmtime(d) <= os.path.getmtime(PREP_LIB_PATH) for d in (PREP_SRC, hdr)):
        return PREP_LIB_PATH
    os.makedirs(LIB_DIR, exist_ok=True)
    env = {k: v for k, v in os.environ.items() if k not in ("CC", "CXX")}
    ccbin = ["-ccbin", "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"]
    subprocess.check_call([_nvcc()] + NVCC_FLAGS + ccbin + ["-I", os.path.join(ROOT, "include"), "-shared", "-o", PREP_LIB_PATH, PREP_SRC], env=env)
    return PREP_LIB_PATH


BATCH_SRC = os.path.join(CSRC, "batch", "vgicp_batch.cpp")
BATCH_LIB_PATH = os.path.join(LIB_DIR, "libvgicp_batch_b200.so")


def build_batch(force=False):
    """Batch registration library (include/vgicp_batch_b200.h): host-only C++ over the C ABI, lib/libvgicp_batch_b200.so."""
    build_native(force=False)
    hdrs = [os.path.join(ROOT, "include", "vgicp_batch_b200.h"), os.path.join(ROOT, "include", "vgicp_b200.h"), LIB_PATH]
    if not force and os.path.exists(BATCH_LIB_PATH) and all(os.path.getmtime(d) <= os.path.getmtime(BATCH_LIB_PATH) for d in [BATCH_SRC] + hdrs):
        return BATCH_LIB_PATH
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    env = {k: v for k, v in os.environ.items() if k not in ("CC", "CXX")}
    subprocess.check_call([gxx, "-shared", "-fPIC", "-fvisibility=hidden", "-std=c++17", "-O2", "-Wall", "-pthread", "-I", os.path.join(ROOT, "include"), BATCH_SRC, "-o", BATCH_LIB_PATH,
                           "-L", LIB_DIR, "-Wl,-rpath,$ORIGIN", "-lvgicp_b200"], env=env)
    return BATCH_LIB_PATH


def build_host_cpp(force=False):
    """C++ host side above the C ABI: the pygicp pybind11 module (fast_gicp_b200/lib/pygicp*.so) and the C++ alignment test
    (fast_gicp_b200/lib/gicp_test), both linked against libvgicp_b200.so with an $ORIGIN rpath."""
    import sysconfig

    import pybind11

    build_native(force=False)
    build_prep(force=False)  # pygicp's downsample / align_points run the device-side ApproximateVoxelGrid
    cpp = os.path.join(HERE, "cpp")
    inc = os.path.join(cpp, "include")
    ext = sysconfig.get_config_var("EXT_SUFFIX") or ".so"
    mod = os.path.join(LIB_DIR, "pygicp" + ext)
    exe = os.path.join(LIB_DIR, "gicp_test")
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    env = {k: v for k, v in os.environ.items() if k not in ("CC", "CXX")}
    hdrs = [os.path.join(inc, "fast_gicp_b200", f) for f in os.listdir(os.path.join(inc, "fast_gicp_b200"))] + [os.path.join(ROOT, "include", "vgicp_b200.h"),
                                                                                                                 os.path.join(ROOT, "include", "vgicp_prep_b200.h"), LIB_PATH]

    def stale(out, srcs):
        return force or not os.path.exists(out) or any(os.path.getmtime(x) > os.path.getmtime(out) for x in srcs + hdrs)

    common = ["-std=c++17", "-O2", "-fPIC", "-Wall", "-I", inc, "-L", LIB_DIR, "-Wl,-rpath,$ORIGIN"]
    src_mod = os.path.join(cpp, "pygicp_module.cpp")
    if stale(mod, [src_mod]):
        subprocess.check_call([gxx, "-shared", "-fvisibility=hidden", src_mod, "-o", mod, "-I", pybind11.get_include(), "-I", sysconfig.get_paths()["include"]] + common +
                              ["-lvgicp_b200", "-lvgicp_prep_b200"], env=env)
    src_test = os.path.join(ROOT, "tests", "cpp", "gicp_test.cpp")
    if stale(exe, [src_test]):
        subprocess.check_call([gxx, src_test, "-o", exe] + common + ["-lvgicp_b200"], env=env)
    return mod, exe


if __name__ == "__main__":
    print(build_native(force="--force" in sys.argv, verbose="-v" in sys.argv))
    print(build_host_cpp(force="--force" in sys.argv))
    print(build_prep(force="--force" in sys.argv))
    print(build_batch(force="--force" in sys.argv))
