"""In-tree build of the native runtime (``pytorch_distributed_train_b200/_C.so``).

One shared object, three kinds of translation units:

* torch-free C++ (store, sockets, CPU collectives, bucket planner) — plain ``g++``;
* torch-facing C++ (comm facade, reducer, bindings, CUDA host glue) — ``g++`` with torch headers;
* sm_90a CUDA (collective + compute kernels) — ``nvcc -gencode arch=compute_90a,code=sm_90a
  -lineinfo``; these TUs never include torch headers so they compile in seconds and
  cross-compile on a GPU-less box.

The ``.so`` is written next to the sources, so the package imports straight from the source tree.
Objects are cached under ``build/`` keyed by a content hash of the TU, its flags and every
header in ``csrc/``.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
import sysconfig
import time
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
BUILD = PKG.parent / "build" / "pdt_obj"
OUT = PKG / "_C.so"
STAMP = PKG / "_C.stamp"

CUDA_HOME = os.environ.get("CUDA_HOME", "/usr/local/cuda")
NVCC = os.path.join(CUDA_HOME, "bin", "nvcc")
ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]


def _torch_paths():
    import torch  # noqa: F401  (import cost is paid once per build)
    from torch.utils import cpp_extension as ce

    inc = ce.include_paths()
    lib = ce.library_paths()
    return inc, lib


def _sources():
    cpp, cu = [], []
    for p in sorted(CSRC.rglob("*")):
        if p.suffix == ".cpp":
            cpp.append(p)
        elif p.suffix == ".cu":
            cu.append(p)
    return cpp, cu


def _headers_digest() -> str:
    h = hashlib.sha256()
    for p in sorted(CSRC.rglob("*")):
        if p.suffix in (".h", ".cuh", ".hpp", ".inl"):
            h.update(str(p.relative_to(CSRC)).encode())
            h.update(p.read_bytes())
    return h.hexdigest()


_INC_RE = None


def _deps_digest(src: Path, _cache={}) -> str:
    """Hash of every project header the TU includes (transitively, quoted includes only)."""
    global _INC_RE
    import re

    if _INC_RE is None:
        _INC_RE = re.compile(r'^\s*#\s*include\s+"([^"]+)"', re.M)
    seen, stack = set(), [src]
    while stack:
        f = stack.pop()
        for inc in _INC_RE.findall(f.read_text()):
            for base in (f.parent, CSRC):
                cand = (base / inc).resolve()
                if cand.exists() and cand not in seen:
                    seen.add(cand)
                    stack.append(cand)
                    break
    h = hashlib.sha256()
    for p in sorted(seen):
        if p not in _cache:
            _cache[p] = hashlib.sha256(p.read_bytes()).hexdigest()
        h.update(str(p).encode())
        h.update(_cache[p].encode())
    return h.hexdigest()


def _needs_torch(src: Path) -> bool:
    txt = src.read_text()
    return ("ATen/" in txt) or ("torch/" in txt) or ("c10/" in txt) or ("comm/comm.h" in txt) or ("reducer.h" in txt)


def _run(cmd, what):
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(f"[pdt build] FAILED: {what}\n$ {' '.join(map(str, cmd))}\n{r.stdout}\n{r.stderr}\n")
        raise RuntimeError(f"native build failed: {what}")
    return r.stdout + r.stderr


def build(verbose: bool = False, force: bool = False, ptxas_info: bool = False) -> Path:
    t0 = time.time()
    BUILD.mkdir(parents=True, exist_ok=True)
    cpp, cu = _sources()
    _ = _headers_digest  # (kept for tooling; object keys use per-TU dependency digests)
    tinc, tlib = _torch_paths()
    pyinc = sysconfig.get_paths()["include"]
    common_inc = [f"-I{CSRC}", f"-I{CUDA_HOME}/include"]
    torch_inc = [f"-isystem{p}" for p in tinc] + [f"-isystem{pyinc}"]
    cxx_flags = ["-O2", "-g0", "-std=c++17", "-fPIC", "-fvisibility=hidden", "-Wall", "-Wno-unused-function",
                 "-D_GLIBCXX_USE_CXX11_ABI=1", "-DTORCH_EXTENSION_NAME=_C", "-DTORCH_API_INCLUDE_EXTENSION_H",
                 "-DPDT_WITH_CUDA=1"]
    nvcc_flags = ["-O3", "-std=c++17", "-lineinfo", "--expt-relaxed-constexpr", "--extended-lambda", "-Xcompiler", "-fPIC",
                  "-Xcompiler", "-fvisibility=hidden", "--threads", "2", "-DPDT_WITH_CUDA=1"] + ARCH_FLAGS
    if ptxas_info:
        nvcc_flags += ["-Xptxas", "-v"]

    jobs = []
    for src in cpp:
        use_torch = _needs_torch(src)
        flags = cxx_flags + common_inc + (torch_inc if use_torch else [])
        jobs.append((src, ["g++", "-c", str(src)] + flags))
    for src in cu:
        jobs.append((src, [NVCC, "-c", str(src)] + nvcc_flags + common_inc))

    objs, todo, keys = [], [], []
    for src, cmd in jobs:
        key = hashlib.sha256((src.read_text() + "\0" + " ".join(cmd) + "\0" + _deps_digest(src)).encode()).hexdigest()[:20]
        keys.append(key)
        obj = BUILD / f"{src.relative_to(CSRC).as_posix().replace('/', '__')}.{key}.o"
        objs.append(obj)
    # The stamp travels with the .so, so a copy of the tree that has the library but not the
    # object cache does not rebuild.
    stamp = hashlib.sha256("".join(keys).encode()).hexdigest()
    if not force and OUT.exists() and STAMP.exists() and STAMP.read_text().strip() == stamp:
        if verbose:
            print(f"[pdt build] {OUT} up to date")
        return OUT
    for (src, cmd), obj in zip(jobs, objs):
        if force or not obj.exists():
            todo.append((src, cmd + ["-o", str(obj)], obj))

    def compile_one(item):
        src, cmd, obj = item
        t = time.time()
        out = _run(cmd, f"compile {src.relative_to(CSRC)}")
        if verbose or ptxas_info:
            print(f"[pdt build] {src.relative_to(CSRC)}  {time.time() - t:.1f}s")
            if ptxas_info and out.strip():
                print(out)
        return obj

    if todo:
        with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 2)) as ex:
            list(ex.map(compile_one, todo))
        # drop stale objects of the same TU
        live = {o.name for o in objs}
        for f in BUILD.glob("*.o"):
            if f.name not in live:
                f.unlink()

    if todo or not OUT.exists() or force:
        rpaths = [f"-Wl,-rpath,{p}" for p in tlib] + ["-Wl,-rpath,$ORIGIN"]
        link = (["g++", "-shared", "-o", str(OUT) + ".tmp"] + [str(o) for o in objs] + [f"-L{p}" for p in tlib] +
                # cudart is linked statically (nvcc's default): our kernels register with our own
                # runtime instance and share torch's primary context / stream handles via the driver.
                ["-lc10", "-ltorch_cpu", "-ltorch", "-ltorch_python", "-lc10_cuda", "-ltorch_cuda",
                 f"-L{CUDA_HOME}/lib64", "-lcudart_static", "-lrt", "-ldl", "-lpthread"] + rpaths)
        _run(link, "link _C.so")
        os.replace(str(OUT) + ".tmp", OUT)
    STAMP.write_text(stamp)
    if verbose:
        print(f"[pdt build] {OUT} ready ({len(todo)}/{len(jobs)} TUs rebuilt, {time.time() - t0:.1f}s)")
    return OUT


def clean():
    shutil.rmtree(BUILD, ignore_errors=True)
    if OUT.exists():
        OUT.unlink()


if __name__ == "__main__":
    import argparse

    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    ap.add_argument("--clean", action="store_true")
    ap.add_argument("--ptxas-info", action="store_true", help="print registers/spills/smem per kernel (-Xptxas -v)")
    a = ap.parse_args()
    if a.clean:
        clean()
    build(verbose=True, force=a.force, ptxas_info=a.ptxas_info)
