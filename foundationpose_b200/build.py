"""In-tree build of libfpose.so (sm_90a only).

`python -m foundationpose_b200.build` or `__graft_entry__.build()`.  nvcc cross-compiles without a
GPU; the resulting .so is git-ignored but travels to the GPU box with the snapshot.
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libfpose.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
]


def _sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _stamp():
    h = hashlib.sha256()
    inc = os.path.join(HERE, "..", "include", "fpose.h")
    files = sorted([os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [inc])
    for f in files:
        with open(f, "rb") as fh:
            h.update(f.encode())
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    """Compile every .cu under csrc/ into lib/libfpose.so.  Incremental per translation unit."""
    os.makedirs(LIBDIR, exist_ok=True)
    stamp_file = os.path.join(LIBDIR, "build.stamp")
    stamp = _stamp()
    if not force and os.path.exists(LIB) and os.path.exists(stamp_file):
        if open(stamp_file).read().strip() == stamp:
            return LIB
    if not os.path.exists(NVCC):
        if os.path.exists(LIB):
            # GPU box without nvcc in PATH: use the prebuilt library that travelled with the snapshot
            return LIB
        raise RuntimeError("nvcc not found and no prebuilt libfpose.so")
    objs = []
    procs = []
    for src in _sources():
        obj = os.path.join(LIBDIR, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        cmd = [NVCC] + NVCC_FLAGS + ["-c", src, "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        log.append(f"==== {os.path.basename(src)}\n{out}")
        if p.returncode != 0:
            failed = True
    with open(os.path.join(LIBDIR, "build.log"), "w") as fh:
        fh.write("\n".join(log))
    if failed or verbose:
        sys.stderr.write("\n".join(log))
    if failed:
        raise RuntimeError("nvcc failed; see foundationpose_b200/lib/build.log")
    cmd = [NVCC, "-shared", "-o", LIB] + objs + ["-lcudart", "-Xlinker", "-rpath,/usr/local/cuda/lib64"]
    subprocess.check_call(cmd)
    with open(stamp_file, "w") as fh:
        fh.write(stamp)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
