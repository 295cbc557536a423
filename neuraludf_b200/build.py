"""In-tree build of libnudf.so (nvcc, sm_90a only).  `python -m neuraludf_b200.build` or __graft_entry__.build()."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libnudf.so")
SOURCES = ["capi.cu", "udf_net.cu", "mlp_nets.cu", "ray_kernels.cu", "sampling.cu", "gemm_tc.cu", "blend.cu", "raygen.cu",
           "mesh_udf.cu", "eval_pc.cu", "mesh_clean.cu", "mesh_band.cu", "mesh_sparse.cu",
           "mesh_post.cu", "mesh_cc.cu", "color_loss.cu", "mesh_grad.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def _stale(obj, src):
    if not os.path.exists(obj):
        return True
    t = os.path.getmtime(obj)
    deps = [src] + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    deps.append(os.path.join(HERE, "..", "include", "nudf.h"))
    deps.append(os.path.abspath(__file__))            # the compiler flags: objects built with other flags are stale
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=True):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    objs, procs = [], []
    for s in SOURCES:
        src = os.path.join(CSRC, s)
        if not os.path.exists(src):
            continue
        obj = os.path.join(objdir, s.replace(".cu", ".o"))
        objs.append(obj)
        if force or _stale(obj, src):
            cmd = [nvcc] + NVCC_FLAGS + ["-c", src, "-o", obj]
            if verbose:
                print(" ".join(cmd), flush=True)
            procs.append((s, subprocess.Popen(cmd)))
    for s, p in procs:
        if p.wait() != 0:
            raise RuntimeError("nvcc failed on " + s)
    if procs or not os.path.exists(LIB):
        cmd = [nvcc, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"]
        if verbose:
            print(" ".join(cmd), flush=True)
        subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv)
