"""ORACLE (test infrastructure) — several ControlNets on one UNet call, as diffusers' `MultiControlNetModel.forward`
(diffusers/models/controlnets/multicontrolnet.py) sums them, and the reference's ControlNet inversion loops
(oracle/controlnet_inversion.py) run with such a sum in place of the one net.

`MultiControlNet(nets, scales)` is called the way the reference calls its ControlNet.  It ignores the
`conditioning_scale=1` the reference passes and gives every net its own scale, as diffusers' pipeline does with a
list of scales.  The conditioning arrives as one tensor, the nets' images concatenated along channels, because the
reference's loop slices it by frame; it is cut back into one image per net here.  Then, as diffusers writes it: every
net on its image and scale, the first net's residuals kept, each later net's added sample by sample, the mid-block
residual with `+=`.
"""
from __future__ import annotations

from typing import Sequence

import torch

from oracle import controlnet_inversion as CI


class MultiControlNet:
    def __init__(self, nets: Sequence, scales: Sequence[float]):
        self.nets, self.scales = list(nets), [float(s) for s in scales]
        assert len(self.nets) == len(self.scales)

    def __call__(self, sample, timestep, encoder_hidden_states=None, controlnet_cond=None, conditioning_scale=1,
                 return_dict=False):
        images = [controlnet_cond[:, 3 * i:3 * i + 3] for i in range(len(self.nets))]
        assert controlnet_cond.shape[1] == 3 * len(self.nets)
        for i, (image, scale, controlnet) in enumerate(zip(images, self.scales, self.nets)):
            down_samples, mid_sample = controlnet(
                sample=sample,
                timestep=timestep,
                encoder_hidden_states=encoder_hidden_states,
                controlnet_cond=image,
                conditioning_scale=scale,
                return_dict=False,
            )
            if i == 0:
                down_block_res_samples, mid_block_res_sample = down_samples, mid_sample
            else:
                down_block_res_samples = [
                    samples_prev + samples_curr
                    for samples_prev, samples_curr in zip(down_block_res_samples, down_samples)
                ]
                mid_block_res_sample += mid_sample
        return down_block_res_samples, mid_block_res_sample


def controlnet_pred(nets, scales, unet, latent_model_input, t, text_embed_input, controlnet_cond):
    """The reference's `controlnet_pred` with the nets' summed residuals."""
    return CI.controlnet_pred(MultiControlNet(nets, scales), unet, latent_model_input, t, text_embed_input,
                              controlnet_cond)


def ddim_inversion(unet, nets, scales, scheduler, cond, controlnet_cond, latent_frames, batch_size, **kw):
    """oracle/controlnet_inversion.py's `ddim_inversion` with the nets' summed residuals; `controlnet_cond` is
    [N, 3K, H, W]."""
    return CI.ddim_inversion(unet, MultiControlNet(nets, scales), scheduler, cond, controlnet_cond, latent_frames,
                             batch_size, **kw)


def ddim_sample(unet, nets, scales, scheduler, x, cond, controlnet_cond, batch_size, **kw):
    """oracle/controlnet_inversion.py's `ddim_sample` with the nets' summed residuals."""
    return CI.ddim_sample(unet, MultiControlNet(nets, scales), scheduler, x, cond, controlnet_cond, batch_size, **kw)
