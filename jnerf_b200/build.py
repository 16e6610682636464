"""Builds libngp_b200.so (all CUDA kernels + the C ABI of include/ngp_b200.h) in-tree with nvcc for sm_90a (H100).
No torch headers are involved: the library's boundary is plain C (pointers and sizes)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libngp_b200.so")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
EXTRA = os.environ.get("NGP_NVCC_FLAGS", "").split()          # extra nvcc flags for experiments
COMMON = EXTRA + ["-O3", "-std=c++17", "-lineinfo", "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC", "-I", os.path.join(HERE, "..", "include")]
# per-file extra flags: the sampler / grid / mesh / render / Mip-NeRF ray code must not contract multiply-adds on its own (bit-exact sample indices)
SOURCES = {
    "capi.cu": [],
    "hash_encode.cu": [],
    "mlp_tc.cu": [],
    "fused_net.cu": [],
    "nerf_mlp.cu": [],
    "mip_mlp.cu": [],
    "mip_sampler.cu": ["-fmad=false"],
    "svox.cu": [],
    "sampler.cu": ["-fmad=false"],
    "grid_update.cu": ["-fmad=false"],
    "mesh.cu": ["-fmad=false"],
    "mesh_smooth.cu": ["-fmad=false"],
    "render.cu": ["-fmad=false"],
    "optimizer.cu": [],
    "compat_tcnn.cu": [],
}


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(HERE, "..", "include", "ngp_b200.h"))
    objs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    procs = []
    for src, extra in SOURCES.items():
        s = os.path.join(CSRC, src)
        o = os.path.join(HERE, "build", src.replace(".cu", ".o"))
        objs.append(o)
        if force or _stale(o, [s] + headers):
            cmd = ["nvcc"] + ARCH + COMMON + extra + (["-Xptxas", "-v"] if verbose else []) + ["-c", s, "-o", o]
            procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            print(f"---- {src} ----\n{out}")
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed")
    if force or procs or _stale(LIB, objs):
        subprocess.check_call(["nvcc"] + ARCH + ["-shared", "-o", LIB] + objs + ["-lcudart_static", "-lpthread", "-ldl", "-lrt"])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
