"""Checks of the stride-2 down-sampler conv (diffusers Downsample2D(padding=0): conv3x3 with stride 2 of
pad(x, (0, 1, 0, 1))) shared by tests/test_vae_encode_cpu.py and tests/test_vae_encode_gpu.py: the fp64 reference, the
per-element bound, the probe inputs, and a torch emulation of the kernel's parity-view addressing (with switchable planted
bugs, so the CPU test can show that the comparator rejects them).

Per-element bound: the kernel multiplies fp16 inputs exactly and accumulates the K = 9 C products and the bias in fp32,
then rounds once to fp16.  Its worst case is (K + 2) 2^-24 (sum_k |x_k w_k| + |b|) for the accumulation plus one fp16
rounding, 2^-11 |y| (2^-25 absolute below the normal range); the comparator allows twice that."""
from __future__ import annotations

import torch
import torch.nn.functional as F

BM = 128
PLANTED = ("symmetric_pad", "view_column_off_by_one", "edge_not_zero_filled", "swapped_parity")


def pick_conv_tile(nimg, H, W):
    """gemm.cu's pick_conv_tile: the 128-pixel TW x TH x TN box with the least padding (ties to the wider TW)."""
    best, best_cost = (1, 1, BM), -1
    tw = 1
    while tw <= BM:
        th = 1
        while tw * th <= BM:
            tn = BM // (tw * th)
            cost = -(-W // tw) * tw * (-(-H // th) * th) * (-(-nimg // tn) * tn)
            if best_cost < 0 or cost < best_cost or (cost == best_cost and tw > best[0]):
                best_cost, best = cost, (tw, th, tn)
            th *= 2
        tw *= 2
    return best


def pack(w):
    """pack_conv3x3's tap-major panel: [Co, Ci, 3, 3] -> [Co, 9 Ci] with column (3 ky + kx) Ci + ci."""
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1).contiguous()


def reference(x16, w16, b):
    """fp64 conv2d(pad(x, (0, 1, 0, 1)), w, stride=2) + b of the fp16 NHWC x [n, H, W, C] -> NHWC [n, H/2, W/2, Co], and
    the matching sum of |x w| + |b| per element."""
    x = x16.double().permute(0, 3, 1, 2)
    w = w16.double()
    bd = b.double()
    ref = F.conv2d(F.pad(x, (0, 1, 0, 1)), w, bd, stride=2).permute(0, 2, 3, 1)
    mag = F.conv2d(F.pad(x.abs(), (0, 1, 0, 1)), w.abs(), bd.abs(), stride=2).permute(0, 2, 3, 1)
    return ref, mag


def bound(ref, mag, K):
    return 2.0 * ((K + 2) * 2.0 ** -24 * mag + 2.0 ** -11 * ref.abs() + 2.0 ** -25)


def compare(out, x16, w16, b):
    """Worst |out - ref| / bound over all elements (<= 1 passes), and the index of the worst element."""
    ref, mag = reference(x16, w16, b)
    assert tuple(out.shape) == tuple(ref.shape), (tuple(out.shape), tuple(ref.shape))
    r = (out.double().to(ref.device) - ref).abs() / bound(ref, mag, 9 * x16.shape[3])
    worst = int(torch.argmax(r.reshape(-1)))
    return float(r.reshape(-1)[worst]), worst


def im2col(x16):
    """Tap-major im2col of the padded stride-2 conv: [n (H/2) (W/2), 9 C], column (3 dy + dx) C + c = x[2y + dy, 2x + dx, c]
    (0 beyond the last row / column)."""
    n, H, W, C = x16.shape
    xp = F.pad(x16, (0, 0, 0, 1, 0, 1))
    cols = [xp[:, dy:dy + H:2, dx:dx + W:2, :] for dy in range(3) for dx in range(3)]
    return torch.cat(cols, -1).reshape(n * (H // 2) * (W // 2), 9 * C)


def _view(x16, py, px, bug):
    """Parity view (py, px) as the TMA descriptor sees it: element (x', y') = input pixel (2 x' + px, 2 y' + py) for
    x' < W / 2, y' < H / 2 and zero fill outside.  Returned padded by one zero row and column, so coordinate W / 2
    (H / 2) reads the fill."""
    n, H, W, C = x16.shape
    Ho, Wo = H // 2, W // 2
    if bug == "edge_not_zero_filled":                 # no fill: the view's addresses run on into the next row / image
        flat = torch.cat([x16.reshape(-1, C), torch.zeros(2 * W + 2, C, dtype=x16.dtype)])
        img = torch.arange(n)[:, None, None]
        yy = torch.arange(Ho + 1)[None, :, None]
        xx = torch.arange(Wo + 1)[None, None, :]
        return flat[img * H * W + (2 * yy + py) * W + 2 * xx + px]
    shift = 1 if (bug == "view_column_off_by_one" and px == 1) else 0
    v = torch.zeros(n, Ho + 1, Wo + 1, C, dtype=x16.dtype)
    src = F.pad(x16, (0, 0, 0, 2))[:, py::2, px + shift::2][:, :Ho, :Wo]
    v[:, :Ho, :src.shape[2]] = src
    return v


def emulate(x16, wp, b, bug=None):
    """The kernel's arithmetic on the CPU: A row (y, x), tap (dy, dx) read from parity view (dy & 1, dx & 1) at
    (x + (dx >> 1), y + (dy >> 1)); fp32 products summed over K, + bias, rounded to fp16.  bug: one of PLANTED."""
    n, H, W, C = x16.shape
    Ho, Wo = H // 2, W // 2
    if bug == "symmetric_pad":                        # the UNet's down-sampler geometry: pad 1 on every side
        xp = F.pad(x16, (0, 0, 1, 1, 1, 1))
        cols = [xp[:, dy:dy + H:2, dx:dx + W:2, :] for dy in range(3) for dx in range(3)]
    else:
        views = {(py, px): _view(x16, py, px, bug) for py in (0, 1) for px in (0, 1)}
        cols = []
        for dy in range(3):
            for dx in range(3):
                py, px = dy & 1, dx & 1
                if bug == "swapped_parity":
                    py, px = px, py
                v = views[(py, px)]
                cols.append(v[:, dy >> 1:(dy >> 1) + Ho, dx >> 1:(dx >> 1) + Wo, :])
    A = torch.cat(cols, -1).reshape(n * Ho * Wo, 9 * C).float()
    out = A @ wp.float().t() + b.float()
    return out.half().reshape(n, Ho, Wo, -1)


def probe_input(n, H, W, C, seed):
    """Sparse impulses (+-1 .. 2, random channels) at the first / last two rows and columns of every image, at the input
    rows / columns around every conv-tile edge of the output grid, and on every image of a tile; zero elsewhere."""
    g = torch.Generator().manual_seed(seed)
    tw, th, tn = pick_conv_tile(n, H // 2, W // 2)
    rows = {0, 1, H - 2, H - 1} | {r for k in range(1, -(-(H // 2) // th)) for r in (2 * k * th - 1, 2 * k * th, 2 * k * th + 1)}
    cols = {0, 1, W - 2, W - 1} | {c for k in range(1, -(-(W // 2) // tw)) for c in (2 * k * tw - 1, 2 * k * tw, 2 * k * tw + 1)}
    x = torch.zeros(n, H, W, C)
    for i in range(n):
        for r in sorted(v for v in rows if 0 <= v < H):
            for c in sorted(v for v in cols if 0 <= v < W):
                ch = torch.randint(0, C, (2,), generator=g)
                x[i, r, c, ch] = (1 + torch.rand(2, generator=g)) * torch.where(torch.rand(2, generator=g) < 0.5, -1.0, 1.0)
    return x.half()


def weights(co, ci, seed):
    g = torch.Generator().manual_seed(seed)
    w = ((torch.rand(co, ci, 3, 3, generator=g) * 2 - 1) / (3 * ci ** 0.5)).half()
    b = 0.1 * torch.randn(co, generator=g)
    return w, b
