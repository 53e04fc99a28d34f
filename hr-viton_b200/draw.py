"""The reference's agnostic masks rasterised on the device (csrc/draw_kernels.cu), pixel for pixel as Pillow 12.2's ImageDraw draws
them: cp_dataset.get_agnostic's bit plane (data.agnostic_bits is its CPU statement) and get_parse_agnostic.get_im_parse_agnostic's
labels.  Keypoints are the (25, 2) OpenPose coordinates as read from the JSON, fp64."""
import numpy as np
import torch

from . import capi

ARM_CANVAS = (768, 1024)  # (w, h): get_agnostic draws its arm masks on this canvas whatever the image size
KEYPOINT_LIMIT = 4096.0  # |coordinate| bound: the ellipse walk's products stay within int64, as in Pillow, well inside it


def keypoints_array(pose, path=""):
    """(25, 2) fp64 keypoints from the reshaped pose_keypoints_2d (K, 2): K >= 13 (get_agnostic reads keypoints 1-12), keypoints
    past 25 dropped and missing ones set absent (0, 0).  Raises ValueError on fewer than 13, or on a coordinate that is not finite
    or beyond +-KEYPOINT_LIMIT."""
    pose = np.asarray(pose, dtype=np.float64)
    if pose.ndim != 2 or pose.shape[1] != 2 or pose.shape[0] < 13:
        raise ValueError("%s: keypoints of shape %s, need (K >= 13, 2)" % (path, pose.shape))
    if not np.isfinite(pose).all() or np.abs(pose).max() > KEYPOINT_LIMIT:
        raise ValueError("%s: a keypoint coordinate is not finite or lies beyond +-%g" % (path, KEYPOINT_LIMIT))
    out = np.zeros((25, 2), np.float64)
    out[:min(25, pose.shape[0])] = pose[:25]
    return out


def _check_keypoints(keypoints):
    if not (torch.is_tensor(keypoints) and keypoints.is_cuda and keypoints.dtype == torch.float64):
        raise ValueError("keypoints: need a CUDA fp64 tensor, got %s" % (keypoints.dtype if torch.is_tensor(keypoints) else type(keypoints)))
    if keypoints.dim() != 3 or tuple(keypoints.shape[1:]) != (25, 2):
        raise ValueError("keypoints: need shape (N, 25, 2), got %s" % (tuple(keypoints.shape),))
    return keypoints.contiguous()


def _workspace(n, h, device, workspace):
    need = capi.lib().hrv_draw_workspace_bytes(n, h)
    if workspace is None or workspace.numel() < need:
        workspace = torch.empty(max(need, 1), dtype=torch.uint8, device=device)
    return workspace


def workspace_bytes(n, h):
    return capi.lib().hrv_draw_workspace_bytes(n, h)


def agnostic_bits(keypoints, out=None, workspace=None):
    """data.agnostic_bits of every sample on the arm canvas: keypoints (N, 25, 2) fp64 CUDA -> (N, 1024, 768) uint8 (into `out`
    when given).  `workspace`: a uint8 CUDA buffer of workspace_bytes(N, 1024) bytes reused across calls (allocated when None)."""
    kp = _check_keypoints(keypoints)
    n, (w, h) = kp.shape[0], ARM_CANVAS
    if out is None:
        out = torch.empty((n, h, w), dtype=torch.uint8, device=kp.device)
    if not (out.is_cuda and out.dtype == torch.uint8 and out.is_contiguous() and tuple(out.shape) == (n, h, w)):
        raise ValueError("out: need a contiguous CUDA uint8 tensor of shape %s" % ((n, h, w),))
    ws = _workspace(n, h, kp.device, workspace)
    capi.check(capi.lib().hrv_agnostic_bits(kp.data_ptr(), n, h, w, out.data_ptr(), ws.data_ptr(), ws.numel(),
                                            torch.cuda.current_stream(kp.device).cuda_stream), "agnostic_bits")
    return out


def parse_agnostic(labels, keypoints):
    """get_im_parse_agnostic(labels, keypoints, w, h) of a batch: labels (N, H, W) uint8 CUDA, keypoints (N, 25, 2) fp64 CUDA ->
    (N, H, W) uint8, the arm masks drawn on the labels' own W x H canvas (the reference's default 768 x 1024 for VITON-HD)."""
    kp = _check_keypoints(keypoints)
    if not (torch.is_tensor(labels) and labels.is_cuda and labels.dtype == torch.uint8 and labels.dim() == 3):
        raise ValueError("labels: need an (N, H, W) CUDA uint8 tensor")
    if labels.shape[0] != kp.shape[0]:
        raise ValueError("labels: %d samples, keypoints: %d" % (labels.shape[0], kp.shape[0]))
    if labels.device != kp.device:
        raise ValueError("labels on %s, keypoints on %s" % (labels.device, kp.device))
    labels = labels.contiguous()
    n, h, w = labels.shape
    out = torch.empty_like(labels)
    ws = _workspace(n, h, kp.device, None)
    capi.check(capi.lib().hrv_parse_agnostic(kp.data_ptr(), labels.data_ptr(), n, h, w, out.data_ptr(), ws.data_ptr(), ws.numel(),
                                             torch.cuda.current_stream(kp.device).cuda_stream), "parse_agnostic")
    return out
