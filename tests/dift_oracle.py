"""TEST INFRASTRUCTURE ONLY.  The DIFT featurizer and read-out restated in torch on the CPU:

  * up_ft: oracle/unet3d_oracle.unet_forward (at any latent size through oracle/sized.py) on a state dict without motion
    modules, read after up block k's up-sampler (up_blocks.k.2 for k = 3, which has none);
  * featurize: the posterior draw and add_noise from given moments and noise, then the ensemble mean of up_ft, fp32;
  * EmulatedReadOut: the read-out kernels' arithmetic (dift.cu) in torch -- bilinear source indices of torch's CPU
    upsample_bilinear2d, the cosine with norms clamped at 1e-8, the frame-order sums -- pluggable into dift.read_out.
"""
from __future__ import annotations

import torch

from oracle import sized as S
from oracle import unet3d_oracle as O


class _Stop(Exception):
    pass


def up_ft(sd, cfg: O.OracleConfig, sample, t, ehs, k: int) -> torch.Tensor:
    """sample [N, 4, 1, h, w] -> up_ft[k] [N, C_k, h_k, w_k] (the forward stops there)."""
    got, taps = {}, {}
    with S.sized_upsampling():
        conv = O._conv_per_frame

        def grab(sd_, p, x, stride=1):
            y = conv(sd_, p, x, stride=stride)
            if p == f"up_blocks.{k}.upsamplers.0.conv":
                got["f"] = y
                raise _Stop
            return y
        O._conv_per_frame = grab
        try:
            O.unet_forward(sd, cfg, sample, t, ehs, taps=taps)
        except _Stop:
            pass
        finally:
            O._conv_per_frame = conv
    f = got["f"] if k < 3 else taps[f"up_blocks.3.{cfg.layers_per_block}"]
    return f[:, :, 0]


def noisy_latents(moments, eps1, eps2, sf, sqrt_a, sqrt_1ma):
    """moments [n, 8, h, w], eps [n E, 4, h, w] -> [n E, 4, 1, h, w] fp32."""
    n = moments.shape[0]
    E = eps1.shape[0] // n
    mu = moments[:, :4].float().repeat_interleave(E, 0)
    std = torch.exp(0.5 * moments[:, 4:].float().clamp(-30.0, 20.0)).repeat_interleave(E, 0)
    z = (mu + std * eps1) * sf
    return (sqrt_a * z + sqrt_1ma * eps2)[:, :, None]


def featurize(sd, cfg, moments, eps1, eps2, sf, sqrt_a, sqrt_1ma, t, ehs1, k):
    """Ensemble means [n, C_k, h_k, w_k] of n frames; ehs1 [1, 77, D] is shared by every member."""
    x = noisy_latents(moments, eps1, eps2, sf, sqrt_a, sqrt_1ma)
    feats = up_ft(sd, cfg, x, t, ehs1.expand(x.shape[0], -1, -1), k)
    n = moments.shape[0]
    return feats.view(n, -1, *feats.shape[1:]).mean(1)


def _src_index(dst, n_in, n_out, align_corners=False):
    d = dst.to(torch.float32)
    if align_corners:
        scale = torch.tensor((n_in - 1) / (n_out - 1) if n_out > 1 else 0.0, dtype=torch.float32)
        s = scale * d
    else:
        scale = torch.tensor(n_in, dtype=torch.float32) / torch.tensor(n_out, dtype=torch.float32)
        s = torch.clamp(scale * (d + 0.5) - 0.5, min=0.0)
    i0 = s.to(torch.int64).clamp(max=n_in - 1)
    i1 = torch.clamp(i0 + 1, max=n_in - 1)
    return i0, i1, s - i0.to(torch.float32)


class EmulatedReadOut:
    """dift.cu's read-out arithmetic on the CPU (the `kernels` argument of videoswap_b200.dift.read_out)."""
    align_corners = False
    count_rejected = False

    @classmethod
    def sample(cls, feat, size, xy):
        """feat NHWC [n, E, h, w, C] -> [n, P, C]: mean over E, then h0l (w0l x00 + w1l x01) + h1l (w0l x10 + w1l x11)."""
        feat = feat.float().cpu()
        xy = xy.long().cpu()
        n, E, h, w, C = feat.shape
        m = feat.sum(1) / E if E > 1 else feat[:, 0]
        H, W = size
        y0, y1, ly1 = _src_index(xy[..., 1], h, H, cls.align_corners)
        x0, x1, lx1 = _src_index(xy[..., 0], w, W, cls.align_corners)
        ly0, lx0 = 1.0 - ly1, 1.0 - lx1
        b = torch.arange(n)[:, None]

        def at(yy, xx):
            return m[b, yy, xx]
        t0 = at(y0, x0) * lx0[..., None] + at(y0, x1) * lx1[..., None]
        t1 = at(y1, x0) * lx0[..., None] + at(y1, x1) * lx1[..., None]
        return t0 * ly0[..., None] + t1 * ly1[..., None]

    @staticmethod
    def cosine(vecs, src, src_row):
        a = vecs.double().cpu()
        b = src.double().cpu()[src_row.long().cpu()]
        na = a.norm(dim=-1).clamp_min(1e-8)
        nb = b.norm(dim=-1).clamp_min(1e-8)
        return ((a * b).sum(-1) / (na * nb)).float()

    @classmethod
    def reduce(cls, vecs, accept):
        vecs = vecs.float().cpu()
        acc = accept.cpu().bool()
        if cls.count_rejected:
            acc_count = torch.ones_like(acc)
        else:
            acc_count = acc
        n, P, C = vecs.shape
        sums = torch.zeros((P, C))
        counts = torch.zeros(P)
        for f in range(n):
            sums += torch.where(acc[f, :, None], vecs[f], torch.zeros(()))
            counts += acc_count[f].float()
        means = torch.where(counts[:, None] != 0, sums / counts.clamp_min(1)[:, None], torch.zeros(()))
        return sums, counts, means
