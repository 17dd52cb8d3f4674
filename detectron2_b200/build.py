"""In-tree build of libd2b200.so (hand-written sm_90a kernels behind include/d2b200.h).

Plain nvcc, no torch headers: the library is a C-ABI .so that the Python host binds with ctypes.
    python -m detectron2_b200.build [--force]
The .so and the objects are build products (git-ignored).
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "_obj")
LIB = os.path.join(HERE, "libd2b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC,-fvisibility=hidden", "--expt-relaxed-constexpr",
          "-diag-suppress", "177"]
# per-file extra flags: the bit-exact ops are compiled without FMA contraction (see DESIGN.md)
SOURCES = {
    "abi.cu": [],
    "roi_align.cu": [],
    "paste_masks.cu": ["-fmad=false"],
    "polygon_masks.cu": ["-fmad=false"],
    "nms.cu": ["-fmad=false"],
    "postproc.cu": ["-fmad=false"],
    "match.cu": ["-fmad=false"],
    "sampling.cu": [],
    "keypoints.cu": ["-fmad=false"],
    "panoptic.cu": ["-fmad=false"],
    "sem_seg_loss.cu": ["-fmad=false"],
    "losses.cu": ["-fmad=false"],
    "deform_conv.cu": [],
    "deform_conv_tc.cu": [],
}


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def _compile(name, extra, force):
    src = os.path.join(CSRC, name)
    obj = os.path.join(OBJ, name.replace(".cu", ".o"))
    deps = [src, os.path.join(CSRC, "common.cuh"), os.path.join(CSRC, "tc_common.cuh"),
            os.path.join(CSRC, "deform_conv_tc.cuh"), os.path.join(CSRC, "rotated_iou.cuh"), os.path.join(CSRC, "boxes.cuh"),
            os.path.join(CSRC, "bilinear.cuh"), os.path.join(CSRC, "polygon_raster.cuh"), os.path.join(HERE, "..", "include", "d2b200.h"), __file__]
    if force or _stale(obj, deps):
        cmd = [NVCC] + ARCH + COMMON + extra + ["-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (name, r.stdout, r.stderr))
        return obj, True
    return obj, False


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        res = list(ex.map(lambda kv: _compile(kv[0], kv[1], force), SOURCES.items()))
    objs = [o for o, _ in res]
    if force or any(ch for _, ch in res) or _stale(LIB, objs):
        cmd = [NVCC] + ARCH + ["-shared", "-o", LIB] + objs + ["-Xcompiler", "-fPIC"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
        if verbose:
            print("built", LIB)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
