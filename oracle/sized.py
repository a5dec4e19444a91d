"""TEST INFRASTRUCTURE ONLY.  The oracle (oracle/unet3d_oracle.py) at latent sizes that are not multiples of 8.

The reference's UNet forwards an explicit up-sampling size when H or W is not a multiple of 8 (unet.py:356-364,454-457;
resnet.py:51-56): every up-sampler but the last block's interpolates to the size of the next skip tensor,
F.interpolate(size=(F, H_l, W_l), mode="nearest"), then runs its 3x3 conv.  With level sizes H_(l+1) = ceil(H_l / 2) the
target is 2n or 2n - 1 for an n-row input, and torch's nearest to 2n - 1 is the 2x nearest image without its last row
(tests/test_latent_sizes_cpu.py checks the identity).  The oracle up-samples by 2; inside `sized_upsampling()` each
up-sampler conv gets that 2x image cropped to the skip's size, which is the reference's computation.  At multiples of 8
the crop is empty and nothing changes.
"""
import re
from contextlib import contextmanager

from oracle import unet3d_oracle as O

_UPSAMPLER = re.compile(r"up_blocks\.(\d+)\.upsamplers\.0\.conv$")


def level_sizes(h, w):
    """(H_l, W_l) of the four UNet levels: the stride-2 down-sampler convs give H_(l+1) = ceil(H_l / 2)."""
    sizes = [(h, w)]
    for _ in range(3):
        sizes.append(((sizes[-1][0] + 1) // 2, (sizes[-1][1] + 1) // 2))
    return sizes


@contextmanager
def sized_upsampling():
    """Within the block, O.unet_forward -- and the loops that call it (O.denoise_step, O.denoise_loop, O.invert_loop) --
    up-sample to the size of the next skip tensor, as the reference does at any latent size."""
    fwd, conv = O.unet_forward, O._conv_per_frame
    sizes = []

    def conv_sized(sd, p, x, stride=1):
        m = _UPSAMPLER.match(p)
        if m is not None:                  # up_blocks.i feeds the skips of level 2 - i
            h, w = sizes[-1][2 - int(m.group(1))]
            x = x[..., :h, :w]
        return conv(sd, p, x, stride=stride)

    def unet_forward_sized(sd, cfg, sample, *args, **kwargs):
        sizes.append(level_sizes(sample.shape[-2], sample.shape[-1]))
        try:
            return fwd(sd, cfg, sample, *args, **kwargs)
        finally:
            sizes.pop()

    O.unet_forward, O._conv_per_frame = unet_forward_sized, conv_sized
    try:
        yield
    finally:
        O.unet_forward, O._conv_per_frame = fwd, conv


def unet_forward(sd, cfg, sample, timestep, ehs, residuals=None, taps=None):
    """O.unet_forward at any latent size (arguments as there; residuals [(B F), C_l, H_l, W_l] on level_sizes)."""
    with sized_upsampling():
        return O.unet_forward(sd, cfg, sample, timestep, ehs, residuals, taps=taps)
