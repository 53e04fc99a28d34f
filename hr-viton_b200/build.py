"""Builds libhrviton_sm100.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

Every kernel translation unit is compiled twice: once as is (bf16 activation storage, entry points hrv_<op>) and once with
-DHRV_F16 -Dhrv=hrv_f16 (IEEE fp16 storage, entry points hrv_<op>_f16; csrc/hrv_f16_rename.h).  capi.cu (error text, device
introspection, TMA descriptor encoder) is shared, and so are conv_f32.cu and metrics.cu, which compute in fp32 / fp64 only, and data_kernels.cu, which takes uint8 and writes fp32, and draw_kernels.cu, which rasterises uint8 masks, and
jpeg_kernels.cu, jpeg_encode.cu and png_encode.cu, which are uint8 / fp32 in and bytes out."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "libhrviton_sm100.so")
SHARED = ["capi.cu"]
KERNEL_TUS = ["conv_igemm.cu", "aux_kernels.cu", "norm_bwd.cu", "conv_wgrad.cu", "glue_kernels.cu", "conv_f32.cu", "syncbn.cu", "metrics.cu", "data_kernels.cu",
             "draw_kernels.cu", "jpeg_kernels.cu", "jpeg_encode.cu", "tv_kernels.cu",
             "png_encode.cu"]
SINGLE = ("conv_f32.cu", "metrics.cu", "data_kernels.cu", "draw_kernels.cu", "jpeg_kernels.cu", "jpeg_encode.cu", "png_encode.cu")  # no 16-bit storage: compiled once
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
         "--expt-relaxed-constexpr", "-Xptxas", "-v"]
F16_FLAGS = ["-DHRV_F16", "-Dhrv=hrv_f16"]


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if not f.endswith(".o")] + [os.path.join(PKG, "..", "include", "hrviton_sm100.h"),
                                                                                         os.path.join(PKG, "..", "include", "hrviton_sm100_metrics.h"),
                                                                                         os.path.join(PKG, "..", "include", "hrviton_sm100_data.h"),
                                                                                         os.path.join(PKG, "..", "include", "hrviton_sm100_jpeg.h"),
                                                                                         os.path.join(PKG, "..", "include", "hrviton_sm100_png.h"),
                                                                                         os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def _jobs():
    jobs = [(s, s.replace(".cu", ".o"), []) for s in SHARED]
    for s in KERNEL_TUS:
        if not os.path.exists(os.path.join(CSRC, s)):
            continue
        jobs.append((s, s.replace(".cu", ".o"), []))
        if s not in SINGLE:
            jobs.append((s, s.replace(".cu", "_f16.o"), F16_FLAGS))
    return jobs


def build(force=False, verbose=False):
    if not force and not _stale():
        return LIB

    def compile_one(job):
        src, obj, extra = job
        cmd = [NVCC] + FLAGS + extra + ["-c", os.path.join(CSRC, src), "-o", os.path.join(CSRC, obj)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        return job, r

    jobs = _jobs()
    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        results = list(ex.map(compile_one, jobs))
    for (src, obj, extra), r in results:
        if verbose or r.returncode:
            sys.stderr.write("==== %s %s\n" % (src, " ".join(extra)) + r.stdout + r.stderr)
        if r.returncode:
            raise RuntimeError("nvcc failed on %s %s" % (src, " ".join(extra)))
    objs = [os.path.join(CSRC, j[1]) for j in jobs]
    r = subprocess.run([NVCC, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"], capture_output=True, text=True)
    if r.returncode:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("link failed")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
