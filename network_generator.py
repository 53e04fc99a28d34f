"""Drop-in for the reference's network_generator.py (network_generator.py:9-433): same public names, constructor /
forward signatures and state_dict keys, backed by the sm_90a kernels of hrviton_b200."""
import hrv_loader

hrv_loader.load()
from hrviton_b200.spade import (BaseNetwork, GANLoss, MaskNorm, MultiscaleDiscriminator, NLayerDiscriminator,  # noqa: E402,F401
                                SPADEGenerator, SPADENorm, SPADEResBlock, get_nonspade_norm_layer)
