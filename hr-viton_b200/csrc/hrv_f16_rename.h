// hrv_f16_rename.h — included (before the public header) by the -DHRV_F16 build of the kernel translation units: every entry
// point of include/hrviton_sm100.h gets its fp16-storage twin hrv_<op>_f16 with the same signature (see the header's "Storage flavours").
#pragma once
#define hrv_conv2d_fwd hrv_conv2d_fwd_f16
#define hrv_instnorm_stats hrv_instnorm_stats_f16
#define hrv_instnorm_apply hrv_instnorm_apply_f16
#define hrv_norm_apply_affine hrv_norm_apply_affine_f16
#define hrv_norm_bwd_reduce hrv_norm_bwd_reduce_f16
#define hrv_norm_bwd_apply hrv_norm_bwd_apply_f16
#define hrv_act_bwd_bias hrv_act_bwd_bias_f16
#define hrv_conv2d_wgrad hrv_conv2d_wgrad_f16
#define hrv_nchw_to_nhwc hrv_nchw_to_nhwc_f16
#define hrv_nhwc_to_nchw hrv_nhwc_to_nchw_f16
#define hrv_space_to_depth hrv_space_to_depth_f16
#define hrv_avgpool3s2 hrv_avgpool3s2_f16
#define hrv_bilinear_up2_add hrv_bilinear_up2_add_f16
#define hrv_flow_warp hrv_flow_warp_f16
#define hrv_bilinear_up2_bwd hrv_bilinear_up2_bwd_f16
#define hrv_flow_warp_bwd hrv_flow_warp_bwd_f16
#define hrv_pack_conv_weight hrv_pack_conv_weight_f16
#define hrv_pack_conv_weight_tf32x2 hrv_pack_conv_weight_tf32x2_f16
#define hrv_space_to_depth_bwd hrv_space_to_depth_bwd_f16
#define hrv_maxpool2_fwd hrv_maxpool2_fwd_f16
#define hrv_maxpool2_bwd hrv_maxpool2_bwd_f16
#define hrv_avgpool3s2_bwd hrv_avgpool3s2_bwd_f16
#define hrv_parse_blur_argmax hrv_parse_blur_argmax_f16
#define hrv_im2col hrv_im2col_f16
#define hrv_l1_sum hrv_l1_sum_f16
#define hrv_l1_bwd hrv_l1_bwd_f16
#define hrv_gaussian_blur hrv_gaussian_blur_f16
#define hrv_flow_warp_nchw hrv_flow_warp_nchw_f16
#define hrv_instnorm_stats2 hrv_instnorm_stats2_f16
#define hrv_onehot_u8 hrv_onehot_u8_f16
#define hrv_conv2d_wgrad_workspace_bytes hrv_conv2d_wgrad_workspace_bytes_f16
