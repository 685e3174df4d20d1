"""In-tree build of the native extension ``ops/_C.so`` for sm_90a (H100).

``python -m rlr_b200.ops.build`` (or ``__graft_entry__.build()``): every ``csrc/*.cu`` is compiled by nvcc with
``-gencode arch=compute_90a,code=sm_90a -lineinfo`` (cross-compiles without a GPU), every ``csrc/*.cpp`` by g++
against the torch headers, and the objects are linked into ``ops/_C.so``.  The .so is git-ignored; nothing is
JIT-compiled at run time.  Objects are rebuilt only when the source or a header changed (content hash), so iterating
on one kernel costs seconds.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "_build")
TARGET = os.path.join(HERE, "_C.so")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def _torch_paths():
    import torch
    from torch.utils import cpp_extension as ce

    inc = ce.include_paths("cuda") if hasattr(ce, "include_paths") else []
    lib = os.path.join(os.path.dirname(torch.__file__), "lib")
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    return inc, lib, abi


def _hash(paths, extra=""):
    """Content hash that is independent of where the repository lives (include / library paths are left out)."""
    h = hashlib.sha256(" ".join(a for a in extra.split() if not a.startswith(("-I", "-L"))).encode())
    for p in sorted(paths, key=os.path.basename):
        with open(p, "rb") as f:
            h.update(os.path.basename(p).encode()); h.update(f.read())
    return h.hexdigest()


def _run(cmd):
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("build failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
    return r.stdout + r.stderr


def build(verbose: bool = False, force: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    inc, torch_lib, abi = _torch_paths()
    py_inc = sysconfig.get_paths()["include"]
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    cu = sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))
    cpp = sorted(f for f in os.listdir(CSRC) if f.endswith(".cpp"))
    inc_flags = [f"-I{p}" for p in [CSRC, py_inc, *inc]]
    nvcc_flags = [*ARCH, "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
                  "-Xptxas", "-v", f"-I{CSRC}", "-I/usr/local/cuda/include"]
    cxx_flags = ["-O2", "-std=c++17", "-fPIC", f"-D_GLIBCXX_USE_CXX11_ABI={abi}", "-DTORCH_EXTENSION_NAME=_C",
                 "-DTORCH_API_INCLUDE_EXTENSION_H", "-Wno-attributes", *inc_flags]
    jobs, objs, logs = [], [], {}

    def need(src, obj, flags):
        stamp = obj + ".sha"
        want = _hash([os.path.join(CSRC, src), *headers], " ".join(flags))
        if not force and os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == want:
            return None
        return want

    for f in cu:
        obj = os.path.join(OBJ, f + ".o"); objs.append(obj)
        want = need(f, obj, nvcc_flags)
        if want:
            jobs.append((f, [NVCC, *nvcc_flags, "-c", os.path.join(CSRC, f), "-o", obj], obj, want))
    for f in cpp:
        obj = os.path.join(OBJ, f + ".o"); objs.append(obj)
        want = need(f, obj, cxx_flags)
        if want:
            jobs.append((f, ["g++", *cxx_flags, "-c", os.path.join(CSRC, f), "-o", obj], obj, want))

    def do(job):
        name, cmd, obj, want = job
        out = _run(cmd)
        with open(obj + ".sha", "w") as fh:
            fh.write(want)
        logs[name] = out
        return name

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            for name in ex.map(do, jobs):
                if verbose:
                    print(f"[build] compiled {name}")
    for name, out in logs.items():  # keep ptxas -v output (registers, spills, smem) next to the objects
        with open(os.path.join(OBJ, name + ".log"), "w") as fh:
            fh.write(out)
    if jobs or force or not os.path.exists(TARGET):
        tmp = TARGET + ".tmp"       # link to a temporary name and rename: a concurrent reader never sees half a file
        link = ["g++", "-shared", "-o", tmp, *objs, f"-L{torch_lib}", "-L/usr/local/cuda/lib64",
                "-lc10", "-ltorch_cpu", "-ltorch", "-ltorch_python", "-lc10_cuda", "-ltorch_cuda", "-lcudart",
                f"-Wl,-rpath,{torch_lib}", "-Wl,-rpath,/usr/local/cuda/lib64"]
        _run(link)
        os.replace(tmp, TARGET)
        if verbose:
            print(f"[build] linked {TARGET}")
    return TARGET


if __name__ == "__main__":
    path = build(verbose=True, force="--force" in sys.argv)
    print(path)
