"""Restatement of stage 1's validation metric (train_condition.py:18-36 and the 'warp_grad' composition of :346-356), the oracle of
hrv_seg_iou / metrics.segmentation_iou.  Counts are exact integers; the arithmetic is numpy float32 with every operation rounded
as torch rounds iou_metric's: intersection (int64) + 1e-7 and union (int64 + fp32) - intersection are fp32, and the per-sample terms
are added in sample order starting from 0.  test_seg_iou_cpu.py ties it to the reference's own iou_metric bit for bit."""
import numpy as np
import torch
import torch.nn.functional as F


def compose(fake_segmap, warped_cm):
    """fake_segmap * cloth_mask, cloth_mask = ones with channel 3 = warped_cm (train_condition.py:352-355)."""
    cloth_mask = torch.ones_like(fake_segmap)
    cloth_mask[:, 3:4] = warped_cm
    return fake_segmap * cloth_mask


def counts(y_pred, y_true):
    """(P, L, I) of one sample: predicted (p > 0.5), labelled (== 1), both."""
    pred, lab = y_pred > 0.5, y_true == 1
    return int(pred.sum()), int(lab.sum()), int((pred & lab).sum())


def iou_metric(y_pred_batch, y_true_batch):
    """iou_metric(y_pred_batch, y_true_batch) as np.float32, for y_true in {0, 1}."""
    B = y_pred_batch.shape[0]
    f = np.float32
    iou = f(0)
    for i in range(B):
        P, L, I = counts(y_pred_batch[i], y_true_batch[i])
        term = (f(I) + f(1e-7)) / ((f(P) + f(L)) - f(I) + f(1e-7)) / f(B)
        iou = f(iou + term)
    return iou


def segmentation_iou(fake_segmap, warped_cm, parse):
    """iou_metric(F.softmax(compose(fake_segmap, warped_cm), 1), parse): torch's soft-max on the inputs' device."""
    return iou_metric(F.softmax(compose(fake_segmap, warped_cm), dim=1), parse)


def probabilities(fake_segmap, warped_cm):
    return F.softmax(compose(fake_segmap, warped_cm), dim=1)
