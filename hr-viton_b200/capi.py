"""ctypes binding of include/hrviton_sm100.h.  There is NO CPU fallback: if the shared library is missing
or a call fails, this raises."""
import ctypes
import os

PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(PKG, "libhrviton_sm100.so")

BF16, F32 = 0, 1  # hrv_dtype codes: 0 = the flavour's 16-bit storage type (bf16 for hrv_<op>, IEEE fp16 for hrv_<op>_f16), 1 = fp32
ACT_NONE, ACT_RELU, ACT_LRELU, ACT_TANH = 0, 1, 2, 3
NHWC, NCHW = 0, 1
EPI_LINEAR, EPI_SPADE = 0, 1
RES_ADD, RES_GATE_RELU, RES_GATE_LRELU = 0, 1, 2

EXPORTS = ["hrv_conv2d_fwd", "hrv_instnorm_stats", "hrv_instnorm_stats2", "hrv_instnorm_apply", "hrv_norm_apply_affine", "hrv_norm_bwd_reduce", "hrv_norm_bwd_apply", "hrv_act_bwd_bias", "hrv_conv2d_wgrad", "hrv_conv2d_wgrad_workspace_bytes", "hrv_nchw_to_nhwc", "hrv_nhwc_to_nchw",
           "hrv_space_to_depth", "hrv_avgpool3s2", "hrv_bilinear_up2_add", "hrv_flow_warp", "hrv_bilinear_up2_bwd", "hrv_flow_warp_bwd", "hrv_pack_conv_weight", "hrv_pack_conv_weight_tf32x2", "hrv_space_to_depth_bwd", "hrv_maxpool2_fwd", "hrv_maxpool2_bwd",
           "hrv_avgpool3s2_bwd", "hrv_parse_blur_argmax", "hrv_parse_blur_argmax_cm", "hrv_gaussian_blur", "hrv_flow_warp_nchw", "hrv_onehot_u8",
           "hrv_onehot_u8_lut", "hrv_im2col", "hrv_l1_sum", "hrv_l1_bwd",
           "hrv_instnorm_stats_workspace_bytes", "hrv_instnorm_stats2_workspace_bytes", "hrv_norm_bwd_reduce_workspace_bytes",
           "hrv_norm_bwd_apply_workspace_bytes", "hrv_act_bwd_bias_ordered", "hrv_act_bwd_bias_ordered_workspace_bytes", "hrv_flow_warp_bwd_ordered",
           "hrv_flow_warp_bwd_ordered_workspace_bytes", "hrv_l1_sum_workspace_bytes", "hrv_flow_warp_nchw_bwd", "hrv_flow_warp_nchw_bwd_workspace_bytes",
           "hrv_grad_unscale_check", "hrv_syncbn_combine", "hrv_syncbn_fwd_finalize", "hrv_syncbn_bwd_finalize", "hrv_seg_softmax_cat", "hrv_seg_iou", "hrv_seg_iou_workspace_bytes",
           "hrv_flow_tv", "hrv_flow_tv_bwd", "hrv_flow_tv_workspace_bytes", "hrv_last_error",
           "hrv_version", "hrv_device_sm_count"]
# include/hrviton_sm100_metrics.h: fp32 / fp64 only, one flavour (no _f16 twin)
METRICS_EXPORTS = ["hrv_lpips_input", "hrv_maxpool3s2", "hrv_lpips_dist", "hrv_ssim", "hrv_ssim_workspace_bytes", "hrv_resize_bilinear_nhwc",
                   "hrv_global_avgpool", "hrv_gram_f64", "hrv_gram_f64_workspace_bytes", "hrv_kid_sums", "hrv_resize_bilinear_fid", "hrv_pool3x3s1"]
SSIM_U8, SSIM_F32 = 0, 1
GRAM_F32, GRAM_F64 = 0, 1
FID_SRC_F32_NCHW, FID_SRC_U8_NHWC = 0, 1
POOL3X3_AVG_EXCL_PAD, POOL3X3_MAX = 0, 1
# include/hrviton_sm100_data.h: uint8 in, fp32 out, one flavour (no _f16 twin)
DATA_EXPORTS = ["hrv_pil_resample_pass", "hrv_pil_nearest", "hrv_agnostic_composite", "hrv_viton_assemble", "hrv_draw_workspace_bytes",
                "hrv_agnostic_bits", "hrv_parse_agnostic"]
# include/hrviton_sm100_jpeg.h: uint8 in and out, one flavour (no _f16 twin)
JPEG_EXPORTS = ["hrv_jpeg_huffman", "hrv_jpeg_idct", "hrv_jpeg_color", "hrv_jpeg_encode_bounds", "hrv_jpeg_encode"]
JPEG_SRC_U8_NHWC, JPEG_SRC_F32_NCHW = 0, 1


class Tensor(ctypes.Structure):
    _fields_ = [("ptr", ctypes.c_void_p), ("n", ctypes.c_int32), ("h", ctypes.c_int32), ("w", ctypes.c_int32),
                ("c", ctypes.c_int32), ("pitch", ctypes.c_int32), ("dtype", ctypes.c_int32)]


class TvFlow(ctypes.Structure):
    _fields_ = [("flow", ctypes.c_void_p), ("h", ctypes.c_int32), ("w", ctypes.c_int32), ("edge_weight", ctypes.c_float),
                ("plain_weight", ctypes.c_float)]


TV_MAX_FLOWS = 5  # HRV_TV_MAX_FLOWS


class VitonPlanes(ctypes.Structure):
    _fields_ = [("image", ctypes.c_void_p), ("cloth", ctypes.c_void_p * 2), ("cloth_mask", ctypes.c_void_p * 2), ("pose", ctypes.c_void_p),
                ("densepose", ctypes.c_void_p), ("agnostic", ctypes.c_void_p), ("parse", ctypes.c_void_p)]


class VitonOutputs(ctypes.Structure):
    _fields_ = [("image", ctypes.c_void_p), ("cloth", ctypes.c_void_p * 2), ("cloth_mask", ctypes.c_void_p * 2), ("pose", ctypes.c_void_p),
                ("densepose", ctypes.c_void_p), ("agnostic", ctypes.c_void_p), ("pcm", ctypes.c_void_p), ("parse_cloth", ctypes.c_void_p),
                ("parse_onehot", ctypes.c_void_p)]


class ConvParams(ctypes.Structure):
    _fields_ = [("inp", Tensor), ("wpack", ctypes.c_void_p),
                ("kh", ctypes.c_int32), ("kw", ctypes.c_int32), ("off_y", ctypes.c_int32), ("off_x", ctypes.c_int32),
                ("bk", ctypes.c_int32), ("bn", ctypes.c_int32), ("n_gemm", ctypes.c_int32),
                ("out", Tensor), ("out_layout", ctypes.c_int32), ("epi", ctypes.c_int32), ("act", ctypes.c_int32),
                ("scale", ctypes.c_void_p), ("shift", ctypes.c_void_p),
                ("res", Tensor), ("x0", Tensor), ("x1", Tensor), ("x0_shift", ctypes.c_int32),
                ("mean", ctypes.c_void_p), ("rstd", ctypes.c_void_p), ("noise", ctypes.c_void_p),
                ("noise_scale", ctypes.c_void_p), ("gamma_out", Tensor), ("res_mode", ctypes.c_int32)]


FLAVOURED = [n for n in EXPORTS if n not in ("hrv_last_error", "hrv_version", "hrv_device_sm_count")]
EXPORTS_F16 = [n + "_f16" for n in FLAVOURED]

_lib = None
_lib_f16 = None


class _F16View:
    """The fp16-storage flavour of the library: attribute hrv_<op> resolves to the symbol hrv_<op>_f16."""

    def __init__(self, L):
        self._L = L

    def __getattr__(self, name):
        return getattr(self._L, name + "_f16" if name in FLAVOURED else name)


def lib(dtype=None):
    """ctypes handle of libhrviton_sm100.so.  dtype torch.float16 selects the fp16-storage flavour of every entry point."""
    global _lib, _lib_f16
    if dtype is not None and str(dtype) == "torch.float16":
        if _lib_f16 is None:
            _lib_f16 = _F16View(lib())
        return _lib_f16
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("hrviton_b200: %s is missing — run `python __graft_entry__.py build` (no CPU fallback exists)" % LIB_PATH)
    L = ctypes.CDLL(LIB_PATH)
    L.hrv_last_error.restype = ctypes.c_char_p
    vp, i32, f32, sz = ctypes.c_void_p, ctypes.c_int32, ctypes.c_float, ctypes.c_size_t
    TP = ctypes.POINTER(Tensor)
    L.hrv_conv2d_fwd.argtypes = [ctypes.POINTER(ConvParams), vp]
    L.hrv_instnorm_stats.argtypes = [TP, i32, TP, i32, i32, vp, vp, f32, vp, vp, vp, ctypes.c_size_t, vp]
    L.hrv_instnorm_stats2.argtypes = [TP, i32, TP, i32, i32, vp, vp, vp, vp, f32, vp, vp, vp, vp, vp, ctypes.c_size_t, vp]
    L.hrv_instnorm_apply.argtypes = [TP, vp, vp, i32, TP, vp]
    L.hrv_norm_bwd_reduce.argtypes = [TP, TP, TP, TP, i32, TP, i32, i32, vp, vp, vp, vp, vp, i32, TP, TP, vp, vp, sz, vp]
    L.hrv_norm_apply_affine.argtypes = [TP, vp, vp, vp, vp, TP, i32, TP, vp]
    L.hrv_norm_bwd_apply.argtypes = [TP, TP, i32, i32, i32, i32, i32, vp, vp, vp, vp, vp, vp, TP, vp, vp, sz, vp]
    L.hrv_act_bwd_bias.argtypes = [TP, TP, i32, TP, vp, vp]
    L.hrv_conv2d_wgrad.argtypes = [TP, TP, i32, i32, i32, vp, vp, ctypes.c_size_t, vp]
    L.hrv_conv2d_wgrad_workspace_bytes.argtypes = [TP, TP, i32, i32]
    L.hrv_nchw_to_nhwc.argtypes = [vp, i32, i32, i32, TP, vp]
    L.hrv_nhwc_to_nchw.argtypes = [TP, vp, vp]
    L.hrv_seg_softmax_cat.argtypes = [vp, i32, vp, i32, vp, i32, vp, i32, i32, i32, TP, vp, vp]
    L.hrv_seg_iou.argtypes = [vp, i32, vp, vp, i32, i32, i32, vp, vp, sz, vp]
    L.hrv_seg_iou_workspace_bytes.argtypes = [i32, i32, i32]
    TVP = ctypes.POINTER(TvFlow)
    L.hrv_flow_tv_workspace_bytes.argtypes = [TVP, i32, i32]
    L.hrv_flow_tv.argtypes = [TVP, i32, i32, vp, i32, i32, vp, vp, ctypes.POINTER(vp), vp, sz, vp]
    L.hrv_flow_tv_bwd.argtypes = [TVP, i32, i32, vp, i32, i32, vp, ctypes.POINTER(vp), vp, vp, sz, vp]
    L.hrv_space_to_depth.argtypes = [TP, TP, vp]
    L.hrv_avgpool3s2.argtypes = [TP, TP, vp]
    L.hrv_bilinear_up2_add.argtypes = [TP, TP, TP, vp]
    L.hrv_flow_warp.argtypes = [vp, vp, vp, TP, TP, vp, vp, vp]
    L.hrv_bilinear_up2_bwd.argtypes = [TP, TP, vp]
    L.hrv_space_to_depth_bwd.argtypes = [TP, TP, vp]
    L.hrv_maxpool2_fwd.argtypes = [TP, TP, vp]
    L.hrv_maxpool2_bwd.argtypes = [TP, TP, TP, i32, vp]
    L.hrv_avgpool3s2_bwd.argtypes = [TP, TP, vp]
    L.hrv_parse_blur_argmax.argtypes = [vp, i32, i32, i32, i32, i32, i32, ctypes.POINTER(ctypes.c_int32), i32, vp, vp, ctypes.c_uint32, vp, vp]
    L.hrv_parse_blur_argmax_cm.argtypes = L.hrv_parse_blur_argmax.argtypes[:-1] + [vp, i32, i32, vp]
    L.hrv_onehot_u8.argtypes = [vp, i32, i32, i32, i32, vp, vp]
    L.hrv_onehot_u8_lut.argtypes = [vp, i32, i32, i32, i32, ctypes.POINTER(ctypes.c_uint8), vp, vp]
    L.hrv_gaussian_blur.argtypes = [vp, i32, i32, i32, i32, f32, vp, vp]
    L.hrv_flow_warp_nchw.argtypes = [vp, i32, i32, i32, vp, vp, vp, i32, i32, i32, vp, i32, i32, f32, f32, vp, vp, vp, vp, i32, vp]
    L.hrv_im2col.argtypes = [TP, TP, i32, i32, i32, vp]
    L.hrv_l1_sum.argtypes = [TP, TP, vp, vp, sz, vp]
    L.hrv_l1_bwd.argtypes = [TP, TP, vp, TP, i32, vp]
    L.hrv_pack_conv_weight.argtypes = [vp, vp, i32, i32, i32, i32, i32, vp, vp, i32, i32, vp]
    L.hrv_pack_conv_weight_tf32x2.argtypes = L.hrv_pack_conv_weight.argtypes
    L.hrv_flow_warp_bwd.argtypes = [vp, vp, vp, TP, TP, vp, vp, vp, vp]
    L.hrv_flow_warp_bwd_ordered.argtypes = [vp, vp, vp, TP, TP, vp, vp, vp, vp, sz, vp]
    L.hrv_flow_warp_bwd_ordered_workspace_bytes.argtypes = [TP, TP]
    L.hrv_act_bwd_bias_ordered.argtypes = [TP, TP, i32, TP, vp, vp, sz, vp]
    L.hrv_act_bwd_bias_ordered_workspace_bytes.argtypes = [TP]
    L.hrv_instnorm_stats_workspace_bytes.argtypes = [TP, TP, i32, i32]
    L.hrv_instnorm_stats2_workspace_bytes.argtypes = [TP, TP]
    L.hrv_norm_bwd_reduce_workspace_bytes.argtypes = [TP, TP, i32, i32]
    L.hrv_norm_bwd_apply_workspace_bytes.argtypes = [TP]
    L.hrv_l1_sum_workspace_bytes.argtypes = [TP]
    L.hrv_flow_warp_nchw_bwd.argtypes = [vp, i32, i32, i32, vp, vp, vp, i32, i32, i32, vp, i32, i32, f32, f32, vp, vp, vp, vp, sz, vp]
    L.hrv_flow_warp_nchw_bwd_workspace_bytes.argtypes = [i32, i32, i32, i32]
    L.hrv_grad_unscale_check.argtypes = [vp, i32, vp, vp, vp]
    f64 = ctypes.c_double
    L.hrv_syncbn_combine.argtypes = [vp, i32, i32, i32, f64, vp, vp]
    L.hrv_syncbn_fwd_finalize.argtypes = [vp, i32, i32, i32, f32, f64, vp, vp, vp, vp, vp]
    L.hrv_syncbn_bwd_finalize.argtypes = [vp, i32, i32, vp, vp, vp]
    for name in FLAVOURED:
        twin = getattr(L, name + "_f16")
        twin.argtypes = getattr(L, name).argtypes
    L.hrv_lpips_input.argtypes = [vp, i32, i32, i32, vp, vp, TP, vp]
    L.hrv_maxpool3s2.argtypes = [TP, TP, vp]
    L.hrv_lpips_dist.argtypes = [TP, vp, vp, vp]
    L.hrv_ssim_workspace_bytes.argtypes = [i32, i32, i32]
    L.hrv_ssim.argtypes = [vp, vp, i32, i32, i32, i32, f64, vp, vp, sz, vp]
    i64 = ctypes.c_int64
    L.hrv_resize_bilinear_nhwc.argtypes = [vp, i32, i32, i32, i32, i32, TP, vp]
    L.hrv_global_avgpool.argtypes = [TP, TP, vp]
    L.hrv_gram_f64_workspace_bytes.argtypes = [i32, i32, i32]
    L.hrv_gram_f64.argtypes = [vp, i64, i64, vp, i64, i64, i32, i32, i32, i32, vp, i64, i32, vp, sz, vp]
    L.hrv_kid_sums.argtypes = [vp, vp, vp, i32, i32, vp, vp, i32, i32, f64, vp, vp]
    L.hrv_resize_bilinear_fid.argtypes = [vp, i32, i32, i32, i32, i32, TP, vp]
    L.hrv_pool3x3s1.argtypes = [TP, i32, TP, vp]
    L.hrv_pil_resample_pass.argtypes = [vp, i32, i32, i32, i32, i32, vp, vp, i32, i32, vp, vp]
    L.hrv_pil_nearest.argtypes = [vp, i32, i32, i32, vp, i32, vp, i32, vp, vp, vp]
    L.hrv_agnostic_composite.argtypes = [vp, vp, vp, i32, i32, i32, vp, vp]
    L.hrv_viton_assemble.argtypes = [ctypes.POINTER(VitonPlanes), ctypes.POINTER(VitonOutputs), i32, i32, i32, vp]
    L.hrv_draw_workspace_bytes.argtypes = [i32, i32]
    L.hrv_agnostic_bits.argtypes = [vp, i32, i32, i32, vp, vp, sz, vp]
    L.hrv_parse_agnostic.argtypes = [vp, vp, i32, i32, i32, vp, vp, sz, vp]
    L.hrv_jpeg_huffman.argtypes = [vp, i32, vp, vp, vp, vp, vp]
    L.hrv_jpeg_idct.argtypes = [vp, i32, vp, vp, i32, vp]
    L.hrv_jpeg_color.argtypes = [vp, i32, vp, i32, vp]
    L.hrv_jpeg_encode_bounds.argtypes = [i32, i32, i32, ctypes.POINTER(sz), ctypes.POINTER(sz)]
    L.hrv_jpeg_encode.argtypes = [vp, i32, i32, i32, i32, vp, vp, sz, vp, sz, vp, vp]
    for name in EXPORTS + EXPORTS_F16 + METRICS_EXPORTS + DATA_EXPORTS + JPEG_EXPORTS:
        fn = getattr(L, name)
        if "_workspace_bytes" in name:
            fn.restype = ctypes.c_size_t
        elif name != "hrv_last_error":
            fn.restype = ctypes.c_int
    _lib = L
    return L


def check(rc, what):
    if rc != 0:
        raise RuntimeError("%s failed (%d): %s" % (what, rc, lib().hrv_last_error().decode()))
