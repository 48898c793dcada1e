"""Builds libttb.so (the sm_90a kernel library behind include/ttb.h) in-tree with nvcc."""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libttb.so")
STAMP = LIB + ".stamp"      # content hash of the sources the library was built from (travels with the .so)
SOURCES = ["capi.cu", "gemm.cu", "norm.cu", "attention.cu", "flash_attn.cu", "ar.cu", "ar_step.cu", "misc.cu", "vocoder.cu", "audio.cu", "wav2vec.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "--use_fast_math",
              "-Xcompiler", "-fPIC", "-Xcompiler", "-O3"]


def _source_hash():
    """Hash of every file under csrc/ + the public header + the flags. File times are not used: a copy of the tree
    need not preserve them, and a spurious rebuild costs minutes."""
    h = hashlib.sha256(" ".join(NVCC_FLAGS).encode())
    files = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC))] + [os.path.join(HERE, "..", "include", "ttb.h")]
    for f in files:
        h.update(os.path.basename(f).encode())
        with open(f, "rb") as fh:
            h.update(fh.read())
    return h.hexdigest()


def build(force=False, verbose=False):
    want = _source_hash()
    if not force and os.path.exists(LIB) and os.path.exists(STAMP) and open(STAMP).read().strip() == want:
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for s in SOURCES:
        o = os.path.join(HERE, "build", s.replace(".cu", ".o"))
        objs.append(o)
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", os.path.join(CSRC, s), "-o", o]
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    ok = True
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            sys.stderr.write("==== %s ====\n%s\n" % (s, out))
        ok = ok and p.returncode == 0
    if not ok:
        raise RuntimeError("nvcc failed")
    cmd = [nvcc, "-shared", "-o", LIB + ".tmp"] + objs + ["-lcudart"]
    subprocess.check_call(cmd)
    os.replace(LIB + ".tmp", LIB)          # atomic: a concurrent reader sees the old or the new library
    with open(STAMP + ".tmp", "w") as f:
        f.write(want + "\n")
    os.replace(STAMP + ".tmp", STAMP)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
