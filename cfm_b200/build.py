"""Build libcfm_b200.so in-tree with nvcc for sm_90a (H100; no torch/pybind coupling: plain C ABI).

    python -m cfm_b200.build          # incremental (per-file .o, rebuilt when sources change)
    python -m cfm_b200.build --force
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libcfm_b200.so")
SOURCES = ["api.cu", "sqdist.cu", "sqdist_h3.cu", "sinkhorn.cu", "sinkhorn_v2.cu", "sample.cu", "assign.cu",
           "gather.cu", "flow.cu", "mlp.cu", "mlp_h3.cu", "rk.cu", "ode_small.cu", "train_small.cu",
           "action_train.cu", "cnf_train.cu", "train_tc.cu", "sde_tc.cu", "cnf_tc.cu",
           "grad_tc.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
         "-Xcompiler", "-fPIC,-O3,-Wall", "--expt-relaxed-constexpr", "-Xptxas", "-v"]


def _digest(paths):
    h = hashlib.sha256(" ".join(FLAGS).encode())
    for p in sorted(paths):
        with open(p, "rb") as f:
            h.update(p.encode() + b"\0" + f.read())
    return h.hexdigest()


def _headers():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hs.append(os.path.join(HERE, "..", "include", "cfm_b200.h"))
    return hs


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    hdr = _headers()
    jobs = []
    for src in SOURCES:
        sp = os.path.join(CSRC, src)
        op = os.path.join(OBJ, src.replace(".cu", ".o"))
        stamp = op + ".sha"
        dig = _digest([sp] + hdr)
        if (not force and os.path.exists(op) and os.path.exists(stamp)
                and open(stamp).read() == dig):
            continue
        jobs.append((sp, op, stamp, dig))

    def run(job):
        sp, op, stamp, dig = job
        r = subprocess.run([NVCC] + FLAGS + ["-c", sp, "-o", op], capture_output=True, text=True)
        with open(op + ".log", "w") as f:
            f.write(r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {sp}:\n{r.stdout}\n{r.stderr}")
        with open(stamp, "w") as f:
            f.write(dig)
        return sp, r.stderr

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            for sp, log in ex.map(run, jobs):
                if verbose:
                    print(f"== {os.path.basename(sp)}\n{log}")
    objs = [os.path.join(OBJ, s.replace(".cu", ".o")) for s in SOURCES]
    if jobs or force or not os.path.exists(LIB):
        r = subprocess.run([NVCC, "-shared", "-o", LIB] + objs +
                           ["-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static"],
                           capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv or "--verbose" in sys.argv))
