"""In-tree nvcc build of libpconv_b200.so (sm_90a only).  No torch headers are involved: the library is
plain CUDA C++ behind a C ABI (include/pconv_b200.h); Python binds it with ctypes."""
import fcntl
import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libpconv_b200.so")
STAMP = os.path.join(HERE, "libpconv_b200.stamp")     # fingerprint of the sources the .so was built from (travels with it)
SOURCES = ["api.cu", "conv_tc.cu", "conv_smallco.cu", "conv_k2r.cu", "conv_stem.cu", "conv_generic.cu", "elementwise.cu", "dwconv.cu", "seg_ops.cu", "inpaint_data.cu", "inpaint_loss.cu", "seg_data.cu", "seg_loss.cu", "text_removal.cu"]
HEADERS = ["pcb_common.cuh", "pcb_ptx.cuh", "pcb_tc_epi.cuh", "pil_data.cuh", "pcb_dilate.cuh", os.path.join("..", "..", "include", "pconv_b200.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
              "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr",
              "-cudart", "static"]


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _fingerprint(sources=None):
    """Content hash of everything the library (or the given sources' objects) is built from: sources, headers, flags,
    this file.  mtimes do not survive a snapshot copy to another machine, contents do."""
    h = hashlib.sha256()
    for d in [os.path.join(CSRC, s) for s in (SOURCES if sources is None else sources) + HEADERS] + [os.path.abspath(__file__)]:
        with open(d, "rb") as f:
            h.update(os.path.basename(d).encode() + b"\0" + f.read() + b"\0")
    h.update(" ".join(NVCC_FLAGS + os.environ.get("PCB_EXTRA_NVCC_FLAGS", "").split()).encode())
    return h.hexdigest()


def needs_build():
    """True when the shared library is missing or was built from different sources / flags."""
    if not os.path.exists(LIB):
        return True
    try:
        with open(STAMP) as f:
            return f.read().strip() != _fingerprint()
    except OSError:
        return True


def build(force=False, verbose=False):
    """Compile every .cu for sm_90a and link libpconv_b200.so.  Safe to call from several processes at once (the ranks
    of a data-parallel job): an exclusive file lock serialises them, objects and the library are written to
    process-private temporaries and renamed into place, and the losers of the race find the stamp up to date."""
    if not force and not needs_build():
        return LIB
    bdir = os.path.join(HERE, "build")
    os.makedirs(bdir, exist_ok=True)
    with open(os.path.join(bdir, ".lock"), "w") as lockf:
        fcntl.flock(lockf, fcntl.LOCK_EX)
        try:
            if not force and not needs_build():      # another process built it while we waited
                return LIB
            return _build_locked(bdir, verbose, force)
        finally:
            fcntl.flock(lockf, fcntl.LOCK_UN)


def _build_locked(bdir, verbose, force=False):
    nvcc = _nvcc()
    fp = _fingerprint()
    tag = f".{os.getpid()}.tmp"
    objs, procs = [], []
    stamps = {}
    for s in SOURCES:
        o = os.path.join(bdir, s.replace(".cu", ".o"))
        objs.append(o)
        # incremental: an object whose own fingerprint (source + headers + flags) is unchanged is kept
        stamps[o] = _fingerprint([s])
        try:
            if not force and os.path.exists(o) and open(o + ".stamp").read().strip() == stamps[o]:
                continue
        except OSError:
            pass
        cmd = [nvcc, *NVCC_FLAGS, *os.environ.get("PCB_EXTRA_NVCC_FLAGS", "").split(), "-c", os.path.join(CSRC, s), "-o", o + tag]
        if verbose:
            print(" ".join(cmd))
        procs.append((s, o, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    failed = None
    for s, _o, p in procs:
        out, _ = p.communicate()
        if p.returncode and failed is None:
            failed = f"nvcc failed on {s}:\n{out.decode()}"
        if verbose and out:
            print(out.decode())
    if failed:
        for _s, o, _p in procs:
            if os.path.exists(o + tag):
                os.remove(o + tag)
        raise RuntimeError(failed)
    for _s, o, _p in procs:
        os.replace(o + tag, o)
        with open(o + ".stamp", "w") as f:
            f.write(stamps[o] + "\n")
    cmd = [nvcc, "-shared", "-o", LIB + tag, *objs, "-cudart", "static"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    if r.returncode:
        raise RuntimeError("link failed:\n" + r.stdout.decode())
    os.replace(LIB + tag, LIB)
    with open(STAMP + tag, "w") as f:
        f.write(fp + "\n")
    os.replace(STAMP + tag, STAMP)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
