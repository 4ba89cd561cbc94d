"""Builds the in-tree CUDA library nv_wavenet_b200/lib/libwavenet_infer.so for sm_90a (nvcc, no GPU needed)."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "lib", "libwavenet_infer.so")


def build(verbose=False, jobs=None):
    jobs = jobs or os.cpu_count() or 4
    cmd = ["make", "-C", os.path.join(HERE, "csrc"), f"-j{jobs}", "all"]
    res = subprocess.run(cmd, stdout=None if verbose else subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc build of libwavenet_infer.so failed:\n" + (res.stdout or ""))
    return LIB


if __name__ == "__main__":
    print(build(verbose=True))
