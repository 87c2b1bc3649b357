"""Builds libsleapb200.so (C-ABI, sm_90a) in-tree with nvcc.  No GPU needed to build."""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libsleapb200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-Xptxas", "-v", "--expt-relaxed-constexpr"]
# per-file extra flags: post-processing must not contract multiply-adds (bit-exact parity); the flow kernels neither,
# so that their float steps round like OpenCV's (sb_flow.cu header); nor the tracker, whose float64 similarities
# restate numpy's (sb_track.cu header)
EXTRA = {"sb_post.cu": ["-fmad=false"], "sb_flow.cu": ["-fmad=false"], "sb_track.cu": ["-fmad=false"]}


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _stamp():
    h = hashlib.sha256()
    for f in sorted(os.listdir(CSRC)) + ["../../include/sleap_b200.h"]:
        p = os.path.join(CSRC, f)
        if os.path.isfile(p):
            h.update(f.encode())
            h.update(open(p, "rb").read())
    return h.hexdigest()


def build(force=False, verbose=False):
    stamp_file = os.path.join(HERE, ".build_stamp")
    stamp = _stamp()
    if not force and os.path.exists(LIB) and os.path.exists(stamp_file) and open(stamp_file).read() == stamp:
        return LIB
    objs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    procs = []
    for src in sources():
        obj = os.path.join(HERE, "build", src.replace(".cu", ".o"))
        cmd = [NVCC] + ARCH + COMMON + EXTRA.get(src, []) + ["-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    log = []
    for src, p in procs:
        out, _ = p.communicate()
        log.append(f"==== {src} ====\n{out}")
        if p.returncode != 0:
            sys.stderr.write(out)
            raise RuntimeError(f"nvcc failed on {src}")
    cmd = [NVCC] + ARCH + ["-shared", "-o", LIB] + objs + ["-cudart", "static"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("link failed")
    with open(os.path.join(HERE, "build", "ptxas.log"), "w") as f:
        f.write("\n".join(log))
    open(stamp_file, "w").write(stamp)
    if verbose:
        print("\n".join(log))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
