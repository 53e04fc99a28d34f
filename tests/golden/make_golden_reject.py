"""Generates tests/golden/reject_256x192_b4.npz: discriminator rejection (get_norm_const.py:93-126, test_condition.py:97-123) on
the UNMODIFIED reference's ConditionGenerator, define_D and D_logit (CPU fp32), with the synthetic weights and inputs of
make_golden.py.  Run where the reference checkout exists:

    python tests/golden/make_golden_reject.py

The last-layer biases of the synthetic discriminator are shifted by `d_bias_shift` so that the normalising constant M is positive
and the logits l stay away from 1: score = l/(1-l)/M amplifies an error in l by 1/(1-l)^2, and a fixture sitting on the pole
would test nothing.  The margin min |1 - l| is asserted here (>= 0.2) and stored."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (reference import, options, save; loads the package)
from hrviton_b200 import synth  # noqa: E402


def main():
    torch.set_num_threads(os.cpu_count())
    ref_networks, _ = mg.import_reference()
    import hrv_env
    hrv_env.install()  # numpy aliases and the shims the reference scripts import
    sys.path.insert(0, mg.REF)
    D_logit = __import__("get_norm_const").D_logit
    sys.path.remove(mg.REF)
    seed, n, h, w, shift, composition = 43, 4, 256, 192, 0.3, "warp_grad"
    with torch.no_grad():
        tocg = ref_networks.ConditionGenerator(mg.tocg_opt(), 4, 16, 13, ngf=96, norm_layer=torch.nn.BatchNorm2d).eval()
        sd = tocg.state_dict()
        synth.fill_state_dict(sd, seed)
        tocg.load_state_dict(sd)
        D = ref_networks.define_D(input_nc=33, Ddownx2=True, Ddropout=True, n_layers_D=3, spectral=False, num_D=2).eval()
        sd = D.state_dict()
        synth.fill_state_dict(sd, seed)
        shifted = [k for k in sd if k.endswith(".bias") and sd[k].numel() == 1]
        assert len(shifted) == 2, shifted
        for k in shifted:
            sd[k] += shift
        D.load_state_dict(sd)
        i1, i2 = synth.tocg_inputs(n, h, w, seed)
        label = synth.one_hot(synth.labels((n, h, w), 13, seed, "dseg"), 13)
        _, seg, _, wcm = tocg(mg.tocg_opt(), i1, i2)
        mask = torch.ones_like(seg)
        mask[:, 3:4] = wcm
        fake = D(torch.cat([i1, i2, torch.softmax(seg * mask, 1)], 1))
        real = D(torch.cat([i1, i2, label], 1))
        l_fake, l_real = D_logit(fake), D_logit(real)
    ratios = torch.cat([l_real / (1 - l_real), l_fake / (1 - l_fake)])
    M = float(ratios.max())
    margin = float((1 - torch.cat([l_real, l_fake])).abs().min())
    assert margin >= 0.2 and M > 0, (margin, M)
    mg.save("reject_256x192_b4", seed=seed, shape=[n, h, w], d_bias_shift=shift, composition=composition, margin=margin,
            l_fake=l_fake, l_real=l_real, M=M, score=l_fake / (1 - l_fake) / M,
            **{"fake_d%d" % i: r[-1] for i, r in enumerate(fake)}, **{"real_d%d" % i: r[-1] for i, r in enumerate(real)})


if __name__ == "__main__":
    main()
