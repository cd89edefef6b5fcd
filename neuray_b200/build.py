"""In-tree build of libneuray_b200.so for sm_90a (nvcc cross-compiles without a GPU).

    python -m neuray_b200.build [--force] [--verbose]

The shared library lands next to this file (neuray_b200/libneuray_b200.so): it is git-ignored but travels to the
GPU box with the gpurun snapshot.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libneuray_b200.so")
SOURCES = ["nr_ops.cu", "nr_pack.cu", "nr_point_kernel.cu", "nr_ray_kernel.cu", "nr_tc_test.cu", "nr_train.cu", "nr_tape_gemm.cu", "nr_encoder.cu", "nr_losses.cu", "nr_mvs.cu", "nr_metrics.cu"]
HEADERS = ["nr_common.cuh", "nr_resample.cuh", "nr_tc.cuh", "nr_point_kernel_pm3.cuh", "nr_train_math.cuh", "nr_conv.cuh", "nr_loss_math.cuh", "nr_mvs.cuh", "nr_mvs_graph.cuh", "nr_encoder_graph.cuh", "nr_metrics_math.cuh", os.path.join("..", "..", "include", "neuray_b200.h")]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "--use_fast_math=false",
         "-Xcompiler", "-fPIC", "-Xcompiler", "-O2"]


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(os.path.join(CSRC, f)) > t for f in SOURCES + HEADERS)


def build(force=False, verbose=False):
    if not force and not _stale():
        return LIB
    flags = [f for f in FLAGS if not f.startswith("--use_fast_math")]
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(CSRC, src.replace(".cu", ".o"))
        cmd = [NVCC, *flags, "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd += ["-Xptxas", "-v"]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            print(out)
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}")
    cmd = [NVCC, "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a"]
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
