"""Build the C-ABI shared library (isaac_ros_nvblox_b200/libnvblox_b200.so) for sm_90a (H100).

nvcc cross-compiles without a GPU. -fmad=false / -ffp-contract=off: one IEEE
rounding per operation on both device and host (DESIGN.md "Numerics").
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libnvblox_b200.so")
SOURCES = ["nvb_api.cu", "nvb_view.cu", "nvb_tsdf.cu", "nvb_esdf.cu", "nvb_esdf_wave.cu", "nvb_esdf_wavex.cu", "nvb_util.cu", "nvb_merge.cu", "nvb_color.cu", "nvb_mesh.cu", "nvb_clear.cu", "nvb_ground.cu", "nvb_dynamics.cu", "nvb_query.cu", "nvb_masker.cu", "nvb_map_io.cu", "nvb_scene.cu"]
HEADERS = [os.path.join(CSRC, "nvb_internal.cuh"), os.path.join(CSRC, "nvb_esdf_block.cuh"), os.path.join(CSRC, "nvb_esdf_common.cuh"), os.path.join(CSRC, "nvb_esdf_wave_common.cuh"), os.path.join(CSRC, "nvb_tma.cuh"), os.path.join(CSRC, "nvb_mc_table.h"), os.path.join(ROOT, "include", "nvblox_b200.h")]


def nvcc_path():
    for p in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if p and (os.path.isabs(p) and os.path.exists(p) or not os.path.isabs(p)):
            return p
    return "nvcc"


def needs_build():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(CSRC, s) for s in SOURCES] + HEADERS + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False, out=None, defines=()):
    """Build the library into OUT (or `out`). `out` builds unconditionally: needs_build() compares file times only, so a
    variant built with other `defines` (e.g. NVB_WAVEX_PROF=1) must go to its own path, never over OUT."""
    if out is None and defines:
        raise ValueError("a build with extra defines needs its own output path")
    if out is None and not force and not needs_build():
        return OUT
    target = out or OUT
    cmd = [
        nvcc_path(), "-std=c++17", "-O3", "-lineinfo",
        "-gencode", "arch=compute_90a,code=sm_90a",
        "-fmad=false", "-prec-div=true", "-prec-sqrt=true", "-ftz=false",
        "-ccbin", "/usr/bin/g++",
        "-Xcompiler", "-fPIC,-ffp-contract=off,-fvisibility=hidden,-O2",
        "-I", os.path.join(ROOT, "include"), "-I", CSRC,
        "-shared", "-cudart", "static",
    ] + os.environ.get("NVB_EXTRA_NVCC_FLAGS", "").split() + ["-D" + d for d in defines] + [
        "-o", target,
    ] + [os.path.join(CSRC, s) for s in SOURCES]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
        print(" ".join(cmd))
    subprocess.check_call(cmd)
    return target


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(OUT)
