"""Build the native library (host C++ + sm_90a CUDA) in-tree with nvcc.

    python -m heyoka_b200.build [--force]

Output: heyoka_b200/lib/libheyoka_b200.so (git-ignored). nvcc cross-compiles for sm_90a (H100) without a GPU.
-fmad=false: the only fused multiply-adds are the explicit fma() calls in csrc/recurrences.cuh (see the floating-point contract there).
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(ROOT, "build", "obj")
LIB = os.path.join(LIBDIR, "libheyoka_b200.so")

HOST_SOURCES = ["expression.cpp", "decompose.cpp", "model.cpp", "lower.cpp", "smem_plan.cpp", "nb_plan.cpp", "nn_plan.cpp",
                "capi_host.cpp", "taylor_adaptive_batch.cpp", "var_ode_sys.cpp", "callback.cpp"]
CUDA_SOURCES = ["batch.cu", "nn_inst.cu", "nb1_inst.cu"]
# The cooperative kernel is instantiated per (lanes per thread, max threads per CTA, mode) family, one
# object each (built in parallel).
COOP_FAMILIES = ([(n, m, g) for n in (1, 2, 4) for m in (512, 256) for g in (1, 0)]
                 + [(1, 512, 4), (2, 512, 4), (1, 512, 5), (2, 512, 5)])

# The dedicated N-body kernel: one object per (lanes per team, CTA-wide team) family.
NB_FAMILIES = [(lt, 0) for lt in (1, 2, 4, 8, 16, 32)] + [(1, 1)]

NVCC_ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
CUDA_FLAGS = ["-lineinfo", "-fmad=false", "-Xcompiler", "-fPIC", "-Xptxas", "-v"]
COMMON = ["-std=c++17", "-O3", "-I" + os.path.join(ROOT, "include"), "-I" + CSRC]


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: cannot build heyoka_b200 (there is no CPU fallback)")


def _deps_newer(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def _all_headers():
    hdrs = []
    for base in (CSRC, os.path.join(ROOT, "include")):
        for dp, _, fns in os.walk(base):
            hdrs += [os.path.join(dp, f) for f in fns if f.endswith((".h", ".hpp", ".cuh"))]
    return hdrs


def build(force=False, verbose=True):
    nvcc = _nvcc()
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(OBJDIR, exist_ok=True)
    hdrs = _all_headers()
    srcs = [os.path.join(CSRC, f) for f in HOST_SOURCES + CUDA_SOURCES + ["coop_inst.cu", "nb_inst.cu"]]
    if not force and not _deps_newer(LIB, srcs + hdrs):
        return LIB  # up to date
    jobs = []  # (obj, deps, cmd)
    for src in HOST_SOURCES + CUDA_SOURCES:
        path = os.path.join(CSRC, src)
        obj = os.path.join(OBJDIR, src + ".o")
        if src.endswith(".cu"):
            cmd = [nvcc] + NVCC_ARCH + COMMON + CUDA_FLAGS + ["-c", path, "-o", obj]
        else:
            # -ffp-contract=off: no FMA contraction on hosts whose baseline has FMA (aarch64), so that the host arithmetic
            # shared with the kernels (angle_reduce.hpp) gives their bits.
            cmd = [nvcc] + NVCC_ARCH + COMMON + ["-Xcompiler", "-fPIC,-Wall,-Wextra,-ffp-contract=off", "-c", path, "-o",
                                                 obj]
        jobs.append((obj, path, cmd))
    inst = os.path.join(CSRC, "coop_inst.cu")
    for n_lanes, maxt, gen in COOP_FAMILIES:
        obj = os.path.join(OBJDIR, "coop_inst_n%d_%d_m%d.o" % (n_lanes, maxt, gen))
        cmd = [nvcc] + NVCC_ARCH + COMMON + CUDA_FLAGS + ["-DHY_COOP_N=%d" % n_lanes, "-DHY_COOP_MAXT=%d" % maxt,
                                                          "-DHY_COOP_MODE=%d" % gen, "-c", inst, "-o", obj]
        jobs.append((obj, inst, cmd))
    nb_inst = os.path.join(CSRC, "nb_inst.cu")
    for lt, cta in NB_FAMILIES:
        obj = os.path.join(OBJDIR, "nb_inst_lt%d_cta%d.o" % (lt, cta))
        cmd = [nvcc] + NVCC_ARCH + COMMON + CUDA_FLAGS + ["-DHY_NB_LT=%d" % lt, "-DHY_NB_CTA=%d" % cta, "-c", nb_inst,
                                                          "-o", obj]
        jobs.append((obj, nb_inst, cmd))
    objs = [j[0] for j in jobs]
    # Headers each kind of object depends on (a change in the N-body kernel does not rebuild the cooperative families).
    nb_only = {"nb_kernel.cuh", "nb1_kernel.cuh", "nb_core.hpp", "nb_desc.hpp", "nb_plan.hpp", "nb_variants.hpp", "nn_kernel.cuh", "nn_plan.hpp",
               "nn_variants.hpp"}
    host_only = {"smem_plan.hpp", "capi_common.hpp", "program.hpp"}

    def deps_of(job):
        name = os.path.basename(job[0])
        if name.startswith("coop_inst"):
            return [h for h in hdrs if os.path.basename(h) not in nb_only | host_only
                    and not h.startswith(os.path.join(ROOT, "include", "heyoka_b200") + os.sep)]
        if name.startswith("nb_inst"):
            return [h for h in hdrs if os.path.basename(h) not in host_only | {"nb_plan.hpp", "coop_variants.hpp"}
                    and not h.startswith(os.path.join(ROOT, "include", "heyoka_b200") + os.sep)]
        return hdrs

    todo = [j for j in jobs if force or _deps_newer(j[0], [j[1]] + deps_of(j))]

    def run(job):
        if verbose:
            print(" ".join(job[2]), flush=True)
        res = subprocess.run(job[2], capture_output=True, text=True)
        with open(job[0] + ".log", "w") as f:
            f.write(res.stdout + res.stderr)  # ptxas -v resource usage
        if res.returncode != 0:
            raise RuntimeError("compilation of %s failed:\n%s\n%s" % (job[1], res.stdout, res.stderr))

    if todo:
        from concurrent.futures import ThreadPoolExecutor
        with ThreadPoolExecutor(max_workers=max(1, min(len(todo), os.cpu_count() or 1))) as ex:
            list(ex.map(run, todo))
    rebuilt = bool(todo)
    if rebuilt or not os.path.exists(LIB):
        cmd = [nvcc] + NVCC_ARCH + ["-shared", "-o", LIB] + objs
        if verbose:
            print(" ".join(cmd), flush=True)
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (res.stdout, res.stderr))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
