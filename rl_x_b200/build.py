"""Builds the C-ABI CUDA library in-tree: rl_x_b200/lib/librlx_b200.so (sm_90a only).

    python -m rl_x_b200.build [--force] [--verbose]

nvcc cross-compiles without a GPU.  The .so and the objects are build products and stay out of git.
"""
import hashlib
import os
import subprocess
import sys

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
LIB_DIR = os.path.join(PKG_DIR, "lib")
LIB_PATH = os.path.join(LIB_DIR, "librlx_b200.so")
STAMP = os.path.join(LIB_DIR, "librlx_b200.stamp")
INCLUDE = os.path.join(os.path.dirname(PKG_DIR), "include")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC",
]
OBJ_DIR = os.path.join(LIB_DIR, "obj")


def _sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cpp")))


def _headers_digest():
    h = hashlib.sha256()
    files = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h", ".hpp"))) + [os.path.join(INCLUDE, "rlx_b200.h")]
    for f in files:
        h.update(os.path.basename(f).encode())      # names, not absolute paths: the digest must not depend on where the tree is checked out
        with open(f, "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def _digest():
    h = hashlib.sha256()
    h.update(_headers_digest().encode())
    for f in _sources():
        h.update(os.path.basename(f).encode())
        with open(f, "rb") as fh:
            h.update(fh.read())
    return h.hexdigest()


def nvcc_path():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def is_fresh():
    if not (os.path.exists(LIB_PATH) and os.path.exists(STAMP)):
        return False
    with open(STAMP) as fh:
        return fh.read().strip() == _digest()


def _compile_one(src, hdr_digest, verbose):
    """One translation unit -> lib/obj/<name>.o, skipped when the source, every header and the flags are unchanged."""
    name = os.path.splitext(os.path.basename(src))[0]
    obj, stamp = os.path.join(OBJ_DIR, name + ".o"), os.path.join(OBJ_DIR, name + ".stamp")
    h = hashlib.sha256(hdr_digest.encode())
    with open(src, "rb") as fh:
        h.update(fh.read())
    want = h.hexdigest()
    if os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read().strip() == want:
        return obj, None
    tmp = obj + ".tmp%d" % os.getpid()
    cmd = [nvcc_path()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", "-o", tmp, src]
    proc = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    if proc.returncode != 0:
        if os.path.exists(tmp):
            os.remove(tmp)
        return obj, "nvcc failed:\n" + " ".join(cmd) + "\n" + proc.stdout + proc.stderr
    if verbose:
        sys.stderr.write(proc.stderr)
    os.replace(tmp, obj)
    with open(stamp, "w") as fh:
        fh.write(want)
    return obj, None


def build(force=False, verbose=False):
    """Compile every CUDA source for sm_90a (one nvcc process per translation unit, in parallel, unchanged units are reused) and link
    them into one shared library. Returns the path."""
    os.makedirs(OBJ_DIR, exist_ok=True)
    if not force and is_fresh():
        return LIB_PATH
    # One builder at a time: the ranks of a torchrun job all call load() at start-up, and a stale library must be rebuilt by exactly one of
    # them while the others wait and then find it fresh.
    import fcntl
    with open(os.path.join(LIB_DIR, ".build.lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not force and is_fresh():
                return LIB_PATH
            return _build_locked(force, verbose)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)


def _build_locked(force, verbose):
    if force:
        for f in os.listdir(OBJ_DIR):
            os.remove(os.path.join(OBJ_DIR, f))
    from concurrent.futures import ThreadPoolExecutor
    hdr = _headers_digest()
    srcs = _sources()
    with ThreadPoolExecutor(max_workers=min(len(srcs), os.cpu_count() or 4)) as ex:
        results = list(ex.map(lambda s_: _compile_one(s_, hdr, verbose), srcs))
    errors = [e for _, e in results if e]
    if errors:
        raise RuntimeError("\n".join(errors))
    tmp = LIB_PATH + ".tmp%d" % os.getpid()
    cmd = [nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-Xcompiler", "-fPIC", "-o", tmp] + [o for o, _ in results]
    proc = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    if proc.returncode != 0:
        if os.path.exists(tmp):
            os.remove(tmp)
        raise RuntimeError("link failed:\n" + " ".join(cmd) + "\n" + proc.stdout + proc.stderr)
    os.replace(tmp, LIB_PATH)           # a process that already mapped the old file keeps it; nobody ever maps a half-written one
    with open(STAMP, "w") as fh:
        fh.write(_digest())
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
