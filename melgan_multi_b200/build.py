"""In-tree build of libmelgan_b200.so (sm_90a only) with nvcc.  No JIT, no torch extension:
the library is a plain C-ABI shared object loaded through ctypes (melgan_multi_b200/engine.py)."""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libmelgan_b200.so")
# test-only second implementation (fp32 SIMT generator, csrc/testlib): built next to the product library, loaded only by
# tests/test_simt_crosscheck_gpu.py -- never by the package
TEST_LIB = os.path.join(LIBDIR, "libmelgan_b200_simt_test.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC", "-Xcompiler", "-O2", "-shared",
    "-cudart", "static",
]


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: libmelgan_b200.so cannot be built (there is no CPU fallback)")


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def test_sources():
    d = os.path.join(CSRC, "testlib")
    return sorted(os.path.join(d, f) for f in os.listdir(d) if f.endswith(".cu")) + [os.path.join(CSRC, "mg_error.cu")]


def needs_build():
    if not os.path.exists(LIB) or not os.path.exists(TEST_LIB):
        return True
    t = min(os.path.getmtime(LIB), os.path.getmtime(TEST_LIB))
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if not os.path.isdir(os.path.join(CSRC, f))]
    deps += test_sources() + [os.path.join(HERE, "..", "include", "melgan_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def _run(cmd, verbose):
    if verbose:
        cmd.insert(1, "-Xptxas")
        cmd.insert(2, "-v")
        print(" ".join(cmd), flush=True)
    env = dict(os.environ)
    env.pop("CC", None); env.pop("CXX", None)
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env)
    if verbose or out.returncode:
        sys.stdout.write(out.stdout)
    if out.returncode:
        raise RuntimeError("nvcc failed (%d)" % out.returncode)


def build(force=False, verbose=False, extra=()):
    if not force and not needs_build():
        return LIB
    os.makedirs(LIBDIR, exist_ok=True)
    extra = list(extra) + os.environ.get("MG_NVCC_EXTRA", "").split()
    _run([_nvcc()] + NVCC_FLAGS + list(extra) + ["-o", TEST_LIB] + test_sources(), False)
    cmd = [_nvcc()] + NVCC_FLAGS + list(extra) + ["-o", LIB] + sources()
    _run(cmd, verbose)
    return LIB


if __name__ == "__main__":
    build(force=True, verbose="-v" in sys.argv)
    print(LIB)
