"""Build libeuler_b200.so in-tree with nvcc for sm_90a (no torch involved)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
SO = os.path.join(LIBDIR, "libeuler_b200.so")
SOURCES = ["graph.cu", "loader.cu", "sample.cu", "walk.cu", "neighbor.cu", "unique.cu", "full_hop.cu", "mp_ops.cu", "gat.cu", "relation.cu", "dna.cu", "segment.cu", "embedding.cu", "graph_label.cu", "readout.cu", "features.cu", "edges.cu", "layerwise.cu", "shard.cu", "p2p.cu", "capi.cu", "host_abi.cu"]
NVCC_FLAGS = ["-std=c++17", "-O3", "-lineinfo", "-gencode", "arch=compute_90a,code=sm_90a",
              "-Xcompiler", "-fPIC", "-Xcompiler", "-O2", "--expt-relaxed-constexpr"]


def _stale():
    if not os.path.exists(SO):
        return True
    t = os.path.getmtime(SO)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + \
           [os.path.join(HERE, "..", "include", "euler_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not _stale():
        return SO
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        nvcc = "nvcc"
    os.makedirs(LIBDIR, exist_ok=True)
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    procs = []
    objs = []
    for src in SOURCES:
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + \
              ["-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    ok = True
    for cmd, p in procs:
        out = p.communicate()[0].decode()
        if p.returncode != 0 or verbose:
            sys.stderr.write(" ".join(cmd) + "\n" + out + "\n")
        ok &= p.returncode == 0
    if not ok:
        raise RuntimeError("nvcc failed")
    tmp = SO + ".tmp.%d" % os.getpid()      # link beside the target, then rename: a reader never sees a half-written library
    cmd = [nvcc, "-shared", "-o", tmp] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"]
    subprocess.check_call(cmd)
    os.replace(tmp, SO)
    return SO


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
