"""CPU oracle of discriminator rejection (get_norm_const.py:60-126, test_condition.py:103-123), built on hrviton_oracle's
tocg_forward / tocg_d_forward and usable under its storage_rounding.  Test infrastructure only, as the oracle itself; pinned
against the live reference by tests/golden/make_golden_reject.py (reject_256x192_b4.npz, tests/test_rejection_cpu.py)."""
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "oracle"))
import hrviton_oracle as orc  # noqa: E402


def d_logit(preds):
    """get_norm_const.py:60-64: the sum over scales of the last output's mean over (1,2,3), each divided by 2 (hard-coded there:
    the mean over scales only for num_D=2)."""
    score = 0
    for p in preds:
        score = score + p[-1].mean((1, 2, 3)) / 2
    return score


def compose_segmap(seg, warped_cm, composition):
    """test_condition.py:108-117: the cloth channel (3) of the scores times the warped cloth mask ('warp_grad') or its > 0.5
    threshold ('detach')."""
    if composition == "no_composition":
        return seg
    mask = torch.ones_like(seg)
    mask[:, 3:4] = (warped_cm > 0.5).float() if composition == "detach" else warped_cm
    return seg * mask


def rejection(sd_tocg, sd_d, input1, input2, norm_const, composition="warp_grad", num_d=2):
    """Discriminator rejection of a generated condition (test_condition.py:103-123).  Returns (score, l, per-scale logit maps)."""
    _, seg, _, wcm = orc.tocg_forward(sd_tocg, input1, input2)
    third = F.softmax(compose_segmap(seg, wcm, composition), dim=1)
    preds = orc.tocg_d_forward(sd_d, torch.cat([input1, input2, third], 1), num_d=num_d)
    l = d_logit(preds)
    return l / (1 - l) / norm_const, l, [p[-1] for p in preds]
