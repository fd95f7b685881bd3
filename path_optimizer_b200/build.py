"""Builds libpqp.so (the C-ABI shared library with the sm_90a kernels) in-tree with nvcc.

Every .cu under csrc/ is compiled to its own object (in parallel) and the objects are linked into one shared
library: each solve kernel sits in its own translation unit on purpose (csrc/pqp_kernels.h)."""
import os
import subprocess
from concurrent.futures import ThreadPoolExecutor

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIB_PATH = os.environ.get("PQP_LIB_OUT") or os.path.join(_HERE, "libpqp.so")   # PQP_LIB_OUT / PQP_NVCC_EXTRA: A/B builds (diagnostics)
OBJ = os.path.join(_HERE, "_obj" + os.environ.get("PQP_OBJ_SUFFIX", ""))
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-diag-suppress", "550,177"]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _deps():
    inc = os.path.join(os.path.dirname(_HERE), "include")
    return [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(inc, f) for f in os.listdir(inc)]


def is_stale():
    if not os.path.exists(LIB_PATH):
        return True
    return any(os.path.getmtime(d) > os.path.getmtime(LIB_PATH) for d in _deps())


def build(force=False, verbose=False, jobs=None):
    """Compile every .cu under csrc/ for sm_90a and link path_optimizer_b200/libpqp.so."""
    if not force and not is_stale():
        return LIB_PATH
    nvcc = os.environ.get("NVCC", "nvcc")
    os.makedirs(OBJ, exist_ok=True)
    extra = (["-Xptxas", "-v"] if verbose else []) + os.environ.get("PQP_NVCC_EXTRA", "").split()
    newest_header = max(os.path.getmtime(d) for d in _deps() if not d.endswith(".cu"))

    def compile_one(src):
        obj = os.path.join(OBJ, os.path.basename(src)[:-3] + ".o")
        if (not force and os.path.exists(obj) and os.path.getmtime(obj) > os.path.getmtime(src)
                and os.path.getmtime(obj) > newest_header):
            return obj, ""
        r = subprocess.run([nvcc] + NVCC_FLAGS + extra + ["-c", src, "-o", obj], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{r.stdout}\n{r.stderr}")
        return obj, r.stderr
    with ThreadPoolExecutor(max_workers=jobs or min(8, os.cpu_count() or 1)) as ex:
        results = list(ex.map(compile_one, sources()))
    if verbose:
        for _, log in results:
            print(log, end="")
    objs = [o for o, _ in results]
    subprocess.run([nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB_PATH] + objs + ["-ldl"], check=True)
    return LIB_PATH


if __name__ == "__main__":
    print(build(force=True, verbose=True))
