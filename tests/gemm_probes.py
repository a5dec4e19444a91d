"""Per-element probes of the tensor-core GEMM / implicit-GEMM convolution (gemm_tc_kernel) shared by
tests/test_gemm_probes_gpu.py and tests/test_gemm_probes_cpu.py: probe inputs, exact references, the activation bounds,
and a torch emulation of the kernel's addressing and epilogue arithmetic (with switchable planted bugs, so the CPU test
can show what the comparators reject).

Integer-exact products.  A and W hold sparse values in {-1, 0, 1}; bias, row vectors and residuals are small integers or
halves.  Every product and every partial sum is then an integer far below 2^11, which fp32 holds exactly in any
accumulation order, so BLOCK_N, the ring depth, the ping-pong split and the tensor core's internal alignment cannot
change the result: the output must equal the fp64 reference exactly (every reference value is checked to be
representable in fp16).  A wrong k-block, tap, concat boundary, image, parity panel, shifted view, stale ring stage,
row-vector row or column chunk is a nonzero integer somewhere.

One-hot precision probes.  Integers cannot see operand precision, so A also carries full-mantissa fp16 values across the
normal range while weight row n has one non-zero, a full-mantissa fp16 w_n at k = j(n).  The accumulator is then a w,
exact in fp32, and the kernel's epilogue order is reproduced exactly: t = fp32(a w); t = fp32(t + bias); t = fp32(t +
rowvec); y = fp16(t); y = fp16(y + R).  Bias and row vectors have bits below fp16 precision, so a bias rounded to fp16, an
operand rounded to bf16, an fp16 accumulation or a residual added before the rounding changes some output bit.  The
comparison is bit for bit (+0 and -0 identified).  For fp16 operands fp32-then-fp16 rounding equals correctly rounded
fp16 arithmetic, so the fp32 restatement of the residual add reproduces __hadd2.

Activations.  GEGLU and quick-GELU run on the same integer pre-activations and are held to the activations' own claimed
error plus one fp16 rounding (tests/norm_probes.py, tests/clip_probes.py).

A backend is an object with the methods of `Emulator` below: the GPU test wraps videoswap_b200.ops, the CPU test runs
the emulation."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from tests import clip_probes as CP
from tests import norm_probes as NP
from tests.downsample_checks import pick_conv_tile

BM, BK, EPI_COLS, GRANULE = 128, 64, 32, 128
LINEAR, GEGLU, QGELU = 0, 1, 2               # ops.EPI_LINEAR, ops.EPI_GEGLU, ops.EPI_QUICK_GELU
H100_SMS = 132
PLANTED = ("odometer_early", "concat_late", "image_ignored", "panel_py_px_swapped", "third_tap_unshifted",
           "rv_mod_ignored", "ldrv_as_n", "geglu_granule_64", "bias_fp16", "operands_bf16", "kblock_fp16",
           "residual_before_rounding")


def pick_bn(m_tiles, N, num_kb, sms):
    """gemm.cu's pick_bn: the automatic column-tile width."""
    if N <= 64:
        return 64
    best, best_cost = 128, -1
    for bn in (128, 160, 256):
        if bn != 128 and N % bn:
            continue
        waves = -(-(m_tiles * -(-N // bn)) // sms)
        cost = waves * (16 + bn // 8)
        if best_cost < 0 or cost < best_cost or (cost == best_cost and num_kb >= 40):
            best, best_cost = bn, cost
    return best


def num_sms(dev):
    dev = torch.device(dev)
    return torch.cuda.get_device_properties(dev).multi_processor_count if dev.type == "cuda" else H100_SMS


# ---------------------------------------------------------------------------------------------------- inputs
def _gen(seed):
    return torch.Generator().manual_seed(seed)


def ternary(shape, seed, density=0.25):
    """Sparse {-1, 0, 1} fp16: about `density` non-zero."""
    g = _gen(seed)
    nz = torch.rand(shape, generator=g) < density
    sign = torch.where(torch.rand(shape, generator=g) < 0.5, -1.0, 1.0)
    return (nz * sign).half()


def halves(shape, seed, lim=2.0):
    """Multiples of 1/2 in [-lim, lim] (fp32)."""
    g = _gen(seed)
    return torch.randint(int(-2 * lim), int(2 * lim) + 1, shape, generator=g).float() / 2


def full16(shape, seed, emin=-4, emax=4):
    """fp16 with the last mantissa bit set (all 11 significant bits used), exponents emin..emax, random sign."""
    g = _gen(seed)
    m = 1024 + 2 * torch.randint(0, 512, shape, generator=g) + 1
    e = torch.randint(emin, emax + 1, shape, generator=g)
    s = torch.where(torch.rand(shape, generator=g) < 0.5, -1.0, 1.0)
    return (s * m.double() * torch.pow(2.0, e.double() - 10)).half()


def fine32(shape, seed, emin=-6, emax=4):
    """fp32 with random bits in all 24 significant bits (13 of them below fp16 precision)."""
    g = _gen(seed)
    m = (1 << 23) + torch.randint(0, 1 << 23, shape, generator=g)
    e = torch.randint(emin, emax + 1, shape, generator=g)
    s = torch.where(torch.rand(shape, generator=g) < 0.5, -1.0, 1.0)
    return (s * m.double() * torch.pow(2.0, e.double() - 23)).float()


def nan16(shape, dev):
    return torch.full(shape, float("nan"), dtype=torch.float16, device=dev)


def table_slice(rows, N, seed, dev, fine=False):
    """A row-vector table as the UNet passes it: a column slice (32 columns in) of a wider fp32 table."""
    t = (fine32 if fine else halves)((rows, N + 96), seed).to(dev)
    return t[:, 32:32 + N]


def epilogue(t, bias=None, rv=None, R=None):
    """The kernel's epilogue order on the fp32 accumulators t: + bias, + row vector (fp32), fp16, then + residual in fp16."""
    t = t.float()
    if bias is not None:
        t = t + bias.float()
    if rv is not None:
        t = t + rv.float()
    y = t.half()
    if R is not None:
        y = (y.float() + R.float()).half()
    return y


def upsample(x, OH, OW):
    """NHWC nearest up-sampling to OH x OW (out[y, x] = in[y // 2, x // 2])."""
    return x[:, torch.arange(OH, device=x.device) // 2][:, :, torch.arange(OW, device=x.device) // 2]


def conv64(x, w):
    """fp64 conv3x3 (pad 1) of NHWC x with w [co, ci, 3, 3] -> NHWC."""
    return F.conv2d(x.double().permute(0, 3, 1, 2), w.double(), padding=1).permute(0, 2, 3, 1)


# ---------------------------------------------------------------------------------------------------- comparators
def _first(bad):
    idx = torch.nonzero(bad)
    return tuple(idx[0].tolist()) if idx.numel() else None


def exact(out, ref, what, dtype=torch.float16):
    """Integer probes: out must equal the fp64 reference exactly (err = max |out - ref|); `dtype` (the output's) must
    represent every reference value."""
    assert torch.equal(ref.to(dtype).double(), ref.double()), f"{what}: probe premise broken, reference not exact in {dtype}"
    o = out.double()
    bad = ~(o == ref)
    n = int(bad.sum())
    if not n:
        return {"err": 0.0, "tol": 0.0, "ok": True, "what": what}
    err = (o - ref).abs().nan_to_num(math.inf).max().item()
    return {"err": err, "tol": 0.0, "ok": False, "what": f"{what}: {n} elements differ, first at {_first(bad)}"}


def _bits(x):
    b = x.contiguous().view(torch.int16)
    return torch.where(b == -32768, torch.zeros_like(b), b)           # -0 as +0


def bitwise(out, expect, what):
    """One-hot probes: out bit for bit equal to the emulated epilogue (err = max |out - expect|)."""
    bad = _bits(out.half()) != _bits(expect.half())
    n = int(bad.sum())
    if not n:
        return {"err": 0.0, "tol": 0.0, "ok": True, "what": what}
    err = (out.double() - expect.double()).abs().nan_to_num(math.inf).max().item()
    return {"err": err, "tol": 0.0, "ok": False, "what": f"{what}: {n} elements differ, first at {_first(bad)}"}


def untouched(buf, written, what):
    """Everything of the NaN-filled buffer outside the written region is still NaN."""
    keep = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
    keep[written] = False
    return NP.flag(bool(torch.isnan(buf[keep]).all()), f"{what}: written outside the output")


def merge(*rs):
    r = dict(max(rs, key=lambda x: x["err"]))
    r["ok"] = all(x["ok"] for x in rs)
    bad = [x for x in rs if not x["ok"]]
    if bad:
        r["what"] = bad[0]["what"]
    return r


def ln_sums_exact(out, sums, bw, what):
    """Row-statistics slices: bit-exact against fp64 sums of the stored fp16 values (exact in fp32 at these sizes)."""
    x = out.double()
    rs = []
    for j in range(-(-x.shape[1] // bw)):
        xs = x[:, j * bw:(j + 1) * bw]
        s, q = xs.sum(1), (xs * xs).sum(1)
        got = sums[j].double()
        rs.append(exact(got[:, 0], s, f"{what} slice {j} sum", torch.float32))
        rs.append(exact(got[:, 1], q, f"{what} slice {j} sum of squares", torch.float32))
    return merge(*rs)


def geglu_bound(v, g):
    """|out - v gelu(g)| bound: gelu_sig's claim |v| (1.2e-5 + 2^-20 max(g, 0)), the fp32 products, one fp16 rounding."""
    y = v * 0.5 * g * (1 + torch.erf(g / math.sqrt(2)))
    e = v.abs() * (NP.GELU_ABS + NP.GELU_REL * g.clamp_min(0)) + 2 * NP.U * y.abs()
    return y, e * (1 + NP.HALF) + NP.HALF * y.abs() + NP.SUB


# ---------------------------------------------------------------------------------------------------- emulation
def pack_conv3x3(w):
    """pack_conv3x3: [Co, Ci, 3, 3] -> [Co, 9 Ci], column (3 ky + kx) Ci + ci."""
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1).contiguous()


def _rng(par, t):
    """Rows (columns) of the 3x3 kernel that sub-pixel tap t of parity `par` gathers: par 0: {0}, {1, 2}; par 1: {0, 1}, {2}."""
    return (0, 0) if (par == 0 and t == 0) else (1, 2) if par == 0 else (0, 1) if t == 0 else (2, 2)


def pack_conv_subpixel(w, odd=False):
    """pack_conv_subpixel: the 4 even panels [4, Co, 4 Ci] (fp32 sums of the gathered taps, rounded to fp16), followed with
    odd=True by the 4 odd-size panels of 6 taps (3 unsummed taps along the odd axis), all flat."""
    co, ci = w.shape[:2]
    wf = w.float()
    panels = []
    for py in (0, 1):
        for px in (0, 1):
            taps = []
            for ty in (0, 1):
                for tx in (0, 1):
                    (r0, r1), (c0, c1) = _rng(py, ty), _rng(px, tx)
                    taps.append(wf[:, :, r0:r1 + 1, c0:c1 + 1].sum((2, 3)))
            panels.append(torch.cat(taps, 1).half())
    if odd:
        for panel in range(4):
            odd_rows = panel < 2
            py, px = (0, panel) if odd_rows else (panel - 2, 0)
            taps = []
            for t in range(6):
                ty, tx = (t >> 1, t & 1) if odd_rows else (t // 3, t % 3)
                r0, r1 = (ty, ty) if odd_rows else _rng(py, ty)
                c0, c1 = _rng(px, tx) if odd_rows else (tx, tx)
                taps.append(wf[:, :, r0:r1 + 1, c0:c1 + 1].sum((2, 3)))
            panels.append(torch.cat(taps, 1).half())
    return torch.cat([p.reshape(-1) for p in panels])


def subpixel_panel(panels, co, ci, py, px, odd_y, odd_x, swapped=False):
    """gemm.cu's subpixel_panel: the weight panel [Co, taps Ci] of output parity (py, px) inside [3x3 | even | odd] panels."""
    if swapped:
        py, px = px, py
    tap = co * ci
    ty3, tx3 = py == 0 and odd_y, px == 0 and odd_x
    if ty3 and tx3:
        off, nt = 0, 9
    elif ty3:
        off, nt = 9 * tap + (16 + 6 * px) * tap, 6
    elif tx3:
        off, nt = 9 * tap + (28 + 6 * py) * tap, 6
    else:
        off, nt = 9 * tap + (2 * py + px) * 4 * tap, 4
    return panels[off:off + nt * tap].view(co, nt * ci)


def pack_geglu(w, b, gran=GRANULE):
    """pack_geglu: value / gate rows interleaved in `gran`-row granules, bias to fp32."""
    hidden = w.shape[0] // 2
    pr = torch.arange(2 * hidden)
    tile, within = pr // (2 * gran), pr % (2 * gran)
    src = torch.where(within < gran, tile * gran + within, hidden + tile * gran + within - gran).to(w.device)
    return w[src].contiguous(), b[src].float()


def _storage(t):
    """The fp32 storage a (view) tensor reads from, starting at its first element."""
    base = torch.empty(0, dtype=t.dtype, device=t.device).set_(t.untyped_storage())
    return base[t.storage_offset():]


def _aligned(t):
    return t is None or t.data_ptr() % 16 == 0


class Emulator:
    """gemm_tc on the CPU: the producer's k-block / tap odometer and concat split over TMA boxes with zero fill, the
    consumer's tile_pixel over pick_conv_tile's TW x TH x TN boxes, sub-pixel panels and shifted views, the staged and
    direct epilogues.  bug: one of PLANTED (None = the kernel as it should be)."""

    def __init__(self, bug=None, sms=H100_SMS):
        assert bug is None or bug in PLANTED, bug
        self.bug, self.sms = bug, sms

    # -------------------------------------------------------------- packing
    def pack_conv3x3(self, w):
        return pack_conv3x3(w)

    def pack_conv_subpixel(self, w):
        return pack_conv_subpixel(w).view(4, w.shape[0], 4 * w.shape[1])

    def pack_geglu(self, w, b):
        return pack_geglu(w, b)

    # -------------------------------------------------------------- entry points
    def gemm(self, A, W, bias=None, A2=None, rowvec=None, ppb=1, rv_mod=0, residual=None, out=None, ln_sums=None, bn=0,
             mode=LINEAR):
        M, N = A.shape[0], W.shape[0]
        if out is None:
            out = torch.empty((M, N // 2 if mode == GEGLU else N), dtype=torch.float16, device=A.device)
        self._tc(A, W, N, out, A2=A2, bias=bias, rowvec=rowvec, ppb=ppb, rv_mod=rv_mod, residual=residual,
                 ln_sums=ln_sums, bn=bn, mode=mode)
        return out

    def conv3x3(self, x, wp, bias=None, x2=None, rowvec=None, ppb=1, rv_mod=0, residual=None, out=None, bn=0):
        n, H, W, _ = x.shape
        co = wp.shape[0]
        if out is None:
            out = torch.empty((n, H, W, co), dtype=torch.float16, device=x.device)
        self._tc(x, wp, co, out.view(-1, co), A2=x2, taps=9, nimg=n, H=H, W=W, bias=bias, rowvec=rowvec, ppb=ppb,
                 rv_mod=rv_mod, residual=None if residual is None else residual.reshape(-1, co), bn=bn)
        return out

    def _upsample(self, x, panels, odd_panels, bias, OH, OW, co):
        n, H, W, ci = x.shape
        out = torch.empty((n, OH, OW, co), dtype=torch.float16, device=x.device)
        for par in range(4):
            py, px = par >> 1, par & 1
            if odd_panels:
                Bw = subpixel_panel(panels, co, ci, py, px, OH & 1, OW & 1, self.bug == "panel_py_px_swapped")
            else:
                q = par if self.bug != "panel_py_px_swapped" else 2 * px + py
                Bw = panels[q]
            self._tc(x, Bw, co, out.view(-1, co), taps=4, nimg=n, H=H, W=W, py=py, px=px, OH=OH, OW=OW, bias=bias)
        return out

    def upsample_sized(self, x, w, bias, OH, OW):
        co, ci = w.shape[:2]
        panels = torch.cat([pack_conv3x3(w).reshape(-1), pack_conv_subpixel(w, odd=True)])
        return self._upsample(x, panels, True, bias, OH, OW, co)

    def upsample_packed(self, x, wsub, bias):
        n, H, W, _ = x.shape
        return self._upsample(x, wsub, False, bias, 2 * H, 2 * W, wsub.shape[1])

    def upsample(self, x, w, bias):
        return self.upsample_packed(x, self.pack_conv_subpixel(w), bias)

    # -------------------------------------------------------------- the kernel
    def _tc(self, A, Bw, N, out, A2=None, taps=1, nimg=0, H=0, W=0, py=0, px=0, OH=0, OW=0, bias=None, rowvec=None,
            ppb=1, rv_mod=0, residual=None, ln_sums=None, bn=0, mode=LINEAR):
        bug, dev = self.bug, A.device
        conv, sub = taps != 1, taps == 4
        K1, K2 = A.shape[-1], 0 if A2 is None else A2.shape[-1]
        ty_n = tx_n = 1
        if sub:
            ty_n, tx_n = (3 if py == 0 and OH % 2 else 2), (3 if px == 0 and OW % 2 else 2)
            ntaps, tap_y0, tap_x0, tap_w, ost, ooy, oox = ty_n * tx_n, py - 1, px - 1, tx_n, 2, py, px
        elif conv:
            ntaps, tap_y0, tap_x0, tap_w, ost, ooy, oox, OH, OW = 9, -1, -1, 3, 1, 0, 0, H, W
        else:
            ntaps = 1
        kb1 = -(-K1 // BK)
        kbt = kb1 + K2 // BK
        nkb = kbt * ntaps
        Ktot = (K1 + K2) * ntaps
        assert tuple(Bw.shape) == (N, Ktot), (tuple(Bw.shape), N, Ktot)
        r = torch.arange(BM, device=dev)
        if conv:
            tw, th, tn = pick_conv_tile(nimg, H, W)
            tiles_x, tiles_y = -(-W // tw), -(-H // th)
            m_tiles = tiles_x * tiles_y * -(-nimg // tn)
            mt = torch.arange(m_tiles, device=dev)
            x0, y0, i0 = (mt % tiles_x) * tw, ((mt // tiles_x) % tiles_y) * th, (mt // (tiles_x * tiles_y)) * tn
            ti, ty, tx = r // (tw * th), (r % (tw * th)) // tw, r % tw
            img = (i0[:, None] + ti[None]).reshape(-1)
            yy = (y0[:, None] + ty[None]).reshape(-1)
            xx = (x0[:, None] + tx[None]).reshape(-1)
        else:
            M = A.shape[0]
            m_tiles = -(-M // BM)
        rows = m_tiles * BM
        gran = 64 if bug == "geglu_granule_64" else GRANULE
        if mode == GEGLU:
            bn = 2 * gran
        elif not bn:
            bn = pick_bn(m_tiles, N, nkb, self.sms)
        n_tiles = -(-N // bn)

        # ---- producer: A operand [rows, nkb * 64] as the TMA boxes deliver it (zero fill outside every view)
        Aop = torch.zeros((rows, nkb * BK), dtype=torch.float16, device=dev)
        for kb in range(nkb):
            rr, tap = kb % kbt, kb // kbt
            if bug == "odometer_early":
                tap = min((kb + 1) // kbt, ntaps - 1)
            first = rr < kb1 + (1 if bug == "concat_late" else 0)
            src = A if first else A2
            c = (rr if first else rr - kb1) * BK
            wdt = max(0, min(BK, src.shape[-1] - c))
            if wdt == 0:
                continue
            if conv:
                dy, dx = tap_y0 + tap // tap_w, tap_x0 + tap % tap_w
                sy = int(ty_n == 3 and dy == tap_y0 + 2 and bug != "third_tap_unshifted")
                sx = int(tx_n == 3 and dx == tap_x0 + 2 and bug != "third_tap_unshifted")
                yv, xv = yy + dy, xx + dx
                ok = (img < nimg) & (yv >= 0) & (yv < H) & (xv >= 0) & (xv < W)
                vals = src[img.clamp(max=nimg - 1), (yv - sy).clamp(0, H - 1), (xv - sx).clamp(0, W - 1), c:c + wdt]
                Aop[:, kb * BK:kb * BK + wdt] = torch.where(ok[:, None], vals, torch.zeros_like(vals))
            else:
                Aop[:M, kb * BK:kb * BK + wdt] = src[:, c:c + wdt]
        Bop = torch.zeros((n_tiles * bn, nkb * BK), dtype=torch.float16, device=dev)
        Bop[:N, :Ktot] = Bw

        # ---- consumers: fp32 accumulation (exact for the probes' data)
        a, b = Aop.double(), Bop.double()
        if bug == "operands_bf16":
            a, b = a.bfloat16().double(), b.bfloat16().double()
        if bug == "kblock_fp16":                          # the last k-block accumulated in fp16
            s = (nkb - 1) * BK
            acc = ((a[:, :s] @ b[:, :s].t()).float() + (a[:, s:] @ b[:, s:].t()).float()).half().float()
        else:
            acc = (a @ b.t()).float()

        # ---- tile_pixel
        if conv:
            im = i0.repeat_interleave(BM) if bug == "image_ignored" else img
            oy, ox = yy * ost + ooy, xx * ost + oox
            valid = (im < nimg) & (yy < H) & (xx < W) & (oy < OH) & (ox < OW)
            pix = (im * OH + oy) * OW + ox
        else:
            pix = torch.arange(rows, device=dev)
            valid = pix < M
        pix, acc = pix[valid], acc[valid]

        # ---- epilogue
        oc = N // 2 if mode == GEGLU else N
        ldrv = N if (rowvec is None or bug == "ldrv_as_n") else rowvec.stride(0)
        staged = (oc % EPI_COLS == 0 and out.stride(0) % 8 == 0 and _aligned(out) and
                  (residual is None or (residual.stride(0) % 8 == 0 and _aligned(residual))) and _aligned(bias) and
                  (rowvec is None or (_aligned(rowvec) and ldrv % 4 == 0)))
        assert staged or mode == LINEAR
        bias32 = None if bias is None else (bias.half().float() if bug == "bias_fp16" else bias.float())
        if mode == GEGLU:
            o = torch.arange(oc, device=dev)
            vcol = (o // gran) * 2 * gran + o % gran
            v, g = acc[:, vcol].double(), acc[:, vcol + gran].double()
            v, g = v + bias32[vcol].double(), g + bias32[vcol + gran].double()
            y = (v * 0.5 * g * (1 + torch.erf(g / math.sqrt(2)))).float().half()
        else:
            t = acc[:, :N]
            if bias32 is not None:
                t = t + bias32
            if rowvec is not None:
                ri = pix // ppb
                if rv_mod > 0 and bug != "rv_mod_ignored":
                    ri = ri % rv_mod
                flat = _storage(rowvec)
                idx = ri[:, None] * ldrv + torch.arange(N, device=dev)[None]
                t = t + torch.where(idx < flat.numel(), flat[idx.clamp(max=flat.numel() - 1)],
                                    torch.full_like(t, float("nan")))
            if mode == QGELU:
                t = CP.quick_gelu64(t).float()
            if residual is not None:
                R = residual[pix].float()
                if not staged and bug == "residual_before_rounding":
                    y = (t + R).half()
                else:
                    y = (t.half().float() + R).half()
            else:
                y = t.half()
        out[pix] = y
        if ln_sums is not None:
            yd = y.double()
            for j in range(n_tiles):
                ys = yd[:, j * bn:(j + 1) * bn]
                ln_sums[j, pix, 0] = ys.sum(1).float()
                ln_sums[j, pix, 1] = (ys * ys).sum(1).float()


# ---------------------------------------------------------------------------------------------------- integer cases
def int_linear(K, dev, M, N, Kd, K2=0, bn=0, rowvec=False, rv_mod=0, residual=None, ln_sums=False, density=0.25,
               seed=0):
    """[A | A2] W^T + bias (+ a row-vector table slice, pix_per_batch 77 or 64 with rv_mod) (+ residual: "sep" or
    "inplace"), written into a view of a NaN-filled buffer (32 columns in, 70 rows spare), optionally with the
    row-statistics slices (NaN-filled, two spare)."""
    A = ternary((M, Kd), seed, density).to(dev)
    A2 = ternary((M, K2), seed + 1, density).to(dev) if K2 else None
    Wt = ternary((N, Kd + K2), seed + 2, density).to(dev)
    b = halves((N,), seed + 3).to(dev)
    ppb = 64 if rv_mod else 77
    rv = table_slice(rv_mod or -(-M // ppb), N, seed + 4, dev) if rowvec else None
    buf = nan16((M + 70, N + 64), dev)
    out = buf[:M, 32:32 + N]
    R = halves((M, N), seed + 5, 4.0).half().to(dev) if residual else None
    if residual == "inplace":
        out.copy_(R)
    ref = A.double() @ Wt[:, :Kd].double().t() + b.double()
    if K2:
        ref = ref + A2.double() @ Wt[:, Kd:].double().t()
    if rowvec:
        ri = torch.arange(M, device=dev) // ppb
        ref = ref + rv.double()[ri % rv_mod if rv_mod else ri]
    if R is not None:
        ref = ref + R.double()
    bw = bn or pick_bn(-(-M // BM), N, -(-Kd // BK) + K2 // BK, num_sms(dev))      # the slices' column width
    nt = -(-N // bw)
    sums = torch.full((nt + 2, M, 2), float("nan"), device=dev) if ln_sums else None
    K.gemm(A, Wt, bias=b, A2=A2, rowvec=rv, ppb=ppb, rv_mod=rv_mod, residual=out if residual == "inplace" else R,
           out=out, ln_sums=sums, bn=bn)
    what = f"gemm M {M} N {N} K {Kd}{f'+{K2}' if K2 else ''} bn {bn or 'auto'}"
    rs = [exact(out, ref, what), untouched(buf, (slice(0, M), slice(32, 32 + N)), what)]
    if ln_sums:
        rs.append(ln_sums_exact(out, sums[:nt], bw, what))
        rs.append(NP.flag(bool(torch.isnan(sums[nt:]).all()), f"{what}: slices past the column tiles written"))
    return merge(*rs)


def int_conv(K, dev, n, H, W, c1, co, c2=0, bn=0, rowvec=False, F_=2, residual=False, density=0.25, seed=0):
    """3x3 conv (+ channel concat) + bias (+ the time-embedding row vector as a table slice, one row per F_ images)
    (+ residual) into the front of a NaN-filled buffer."""
    x1 = ternary((n, H, W, c1), seed, density).to(dev)
    x2 = ternary((n, H, W, c2), seed + 1, density).to(dev) if c2 else None
    w = ternary((co, c1 + c2, 3, 3), seed + 2, density).to(dev)
    b = halves((co,), seed + 3).to(dev)
    rv = table_slice(-(-n // F_), co, seed + 4, dev) if rowvec else None
    R = halves((n, H, W, co), seed + 5, 4.0).half().to(dev) if residual else None
    buf = nan16((n * H * W * co + 4096,), dev)
    out = buf[:n * H * W * co].view(n, H, W, co)
    K.conv3x3(x1, K.pack_conv3x3(w), bias=b, x2=x2, rowvec=rv, ppb=F_ * H * W, residual=R, out=out, bn=bn)
    ref = conv64(x1 if x2 is None else torch.cat([x1, x2], -1), w) + b.double()
    if rowvec:
        ref = ref + rv.double()[torch.arange(n, device=dev) // F_][:, None, None, :]
    if residual:
        ref = ref + R.double()
    what = f"conv {n}x{H}x{W} C {c1}{f'+{c2}' if c2 else ''} -> {co} bn {bn or 'auto'} tile {pick_conv_tile(n, H, W)}"
    return merge(exact(out, ref, what), untouched(buf, slice(0, n * H * W * co), what))


def int_subpixel(K, dev, n, H, W, C, co, OH=0, OW=0, how="sized", seed=0):
    """Nearest up-sampling to OH x OW + conv3x3: "sized" (the UNet's up-sampler, odd sizes too), "packed" (the panels of
    pack_conv_subpixel) or "plain" (upsample_conv3x3); the panels' fp32 tap sums of integers are exact."""
    OH, OW = OH or 2 * H, OW or 2 * W
    x = ternary((n, H, W, C), seed).to(dev)
    w = ternary((co, C, 3, 3), seed + 1, 0.5).to(dev)
    b = halves((co,), seed + 2).to(dev)
    if how == "sized":
        out = K.upsample_sized(x, w, b, OH, OW)
    elif how == "packed":
        out = K.upsample_packed(x, K.pack_conv_subpixel(w), b)
    else:
        out = K.upsample(x, w, b)
    ref = conv64(upsample(x, OH, OW), w) + b.double()
    return exact(out.reshape(n, OH, OW, co), ref, f"up-sampler ({how}) {n}x{H}x{W} -> {OH}x{OW} C {C} -> {co}")


# ---------------------------------------------------------------------------------------------------- one-hot probes
def _one_hot(N, Kd, j, seed, dev):
    W = torch.zeros((N, Kd), dtype=torch.float16)
    w = full16((N,), seed, -3, 3)
    W[torch.arange(N), j] = w
    return W.to(dev), w.to(dev)


def onehot_linear(K, dev, M, Kd, N, bn=0, rowvec=True, rv_mod=0, residual=True, direct=False, seed=0):
    """Weight row n = w_n at k = j(n); j covers every k of the problem over ceil(K / N) launches.  direct: the output is
    8 bytes off a 16-byte boundary, which sends the kernel to its direct-store epilogue."""
    A = full16((M, Kd), seed).to(dev)
    b = fine32((N,), seed + 1).to(dev)
    ppb = 64 if rv_mod else 77
    rv = table_slice(rv_mod or -(-M // ppb), N, seed + 2, dev, fine=True) if rowvec else None
    R = full16((M, N), seed + 3, -3, 3).to(dev) if residual else None
    ri = torch.arange(M, device=dev) // ppb
    rvr = rv[ri % rv_mod if rv_mod else ri] if rowvec else None
    perm = torch.randperm(Kd, generator=_gen(seed + 4))
    rs = []
    for launch in range(-(-Kd // N)):
        j = perm[(launch * N + torch.arange(N)) % Kd]
        W, w = _one_hot(N, Kd, j, seed + 5 + launch, dev)
        if direct:
            buf = nan16((M, N + 8), dev)
            out = buf[:, 4:4 + N]
        else:
            out = None
        out = K.gemm(A, W, bias=b, rowvec=rv, ppb=ppb, rv_mod=rv_mod, residual=R, out=out, bn=bn)
        expect = epilogue(A[:, j.to(dev)].float() * w.float(), b, rvr, R)
        rs.append(bitwise(out, expect, f"one-hot gemm M {M} K {Kd} N {N} bn {bn or 'auto'}"
                                       f"{' direct' if direct or N % 32 else ''} launch {launch}"))
    return merge(*rs)


def two_term(K, dev, M, Kd, N, bn=0, seed=0):
    """Terms in the first and the last k-block whose sum 1 + s is exact in fp32 but not in fp16; bias -1 leaves s.
    An fp16 accumulation gives 0, a dropped last k-block 0, a dropped first one s - 1."""
    g = _gen(seed)
    A = full16((M, Kd), seed + 1)
    A[:, 0] = 1
    A[:, Kd - 1] = ((2 * torch.randint(0, 128, (M,), generator=g) + 1).double() * 2.0 ** -12).half()
    W = torch.zeros((N, Kd), dtype=torch.float16)
    W[:, 0] = 1
    W[:, Kd - 1] = torch.pow(2.0, torch.randint(-1, 2, (N,), generator=g).double()).half()
    b = -torch.ones(N)
    A, W, b = A.to(dev), W.to(dev), b.to(dev)
    out = K.gemm(A, W, bias=b, bn=bn)
    t = (A[:, :1].double() * W[:, 0].double() + A[:, -1:].double() * W[:, -1].double()).float()
    return bitwise(out, epilogue(t, b), f"two-term gemm M {M} K {Kd} N {N} bn {bn or 'auto'}")


def onehot_conv(K, dev, n, H, W, C, residual=True, seed=0):
    """N = 9 C output channels, channel n = one (tap, input channel) of the panel: every tap reads exactly its neighbour,
    or exactly zero from the fill at the image borders."""
    N = 9 * C
    x = full16((n, H, W, C), seed).to(dev)
    perm = torch.randperm(N, generator=_gen(seed + 1))
    w3 = torch.zeros((N, C, 3, 3), dtype=torch.float16)
    w = full16((N,), seed + 2, -3, 3)
    tap, ch = perm // C, perm % C
    w3[torch.arange(N), ch, tap // 3, tap % 3] = w
    w3 = w3.to(dev)
    b = fine32((N,), seed + 3).to(dev)
    R = full16((n, H, W, N), seed + 4, -3, 3).to(dev) if residual else None
    out = K.conv3x3(x, K.pack_conv3x3(w3), bias=b, residual=R)
    expect = epilogue(conv64(x, w3).float(), b, None, R)
    return bitwise(out, expect, f"one-hot conv {n}x{H}x{W} C {C} tile {pick_conv_tile(n, H, W)}")


def onehot_subpixel(K, dev, n, H, W, C, OH, OW, seed=0):
    """The sub-pixel conv with one-hot 3x3 weights (a panel tap sums one non-zero, exactly): every tap of every parity,
    including the third tap of an odd axis read through the shifted view."""
    N = 9 * C
    x = full16((n, H, W, C), seed).to(dev)
    perm = torch.randperm(N, generator=_gen(seed + 1))
    w3 = torch.zeros((N, C, 3, 3), dtype=torch.float16)
    tap, ch = perm // C, perm % C
    w3[torch.arange(N), ch, tap // 3, tap % 3] = full16((N,), seed + 2, -3, 3)
    w3 = w3.to(dev)
    b = fine32((N,), seed + 3).to(dev)
    out = K.upsample_sized(x, w3, b, OH, OW)
    expect = epilogue(conv64(upsample(x, OH, OW), w3).float(), b)
    return bitwise(out.reshape(n, OH, OW, N), expect, f"one-hot up-sampler {n}x{H}x{W} -> {OH}x{OW} C {C}")


def subnormal_probe(K, dev, M=256, Kd=64, N=64, seed=0):
    """Rows 0..M/2-1 of A subnormal fp16 (m 2^-24, m odd), the rest normal; one-hot weights 2^2 .. 2^8 with full
    mantissas.  Returns (subnormal rows exact, normal rows exact): a hardware property, recorded, not asserted."""
    g = _gen(seed)
    A = full16((M, Kd), seed + 1)
    A[:M // 2] = ((2 * torch.randint(0, 512, (M // 2, Kd), generator=g) + 1).double() * 2.0 ** -24).half()
    j = torch.randperm(Kd, generator=g)[torch.arange(N) % Kd]
    W = torch.zeros((N, Kd), dtype=torch.float16)
    w = full16((N,), seed + 2, 2, 8)
    W[torch.arange(N), j] = w
    A, W = A.to(dev), W.to(dev)
    out = K.gemm(A, W)
    expect = epilogue(A[:, j.to(dev)].float() * w.to(dev).float())
    return bitwise(out[:M // 2], expect[:M // 2], "subnormal A")["ok"], bitwise(out[M // 2:], expect[M // 2:], "normal A")["ok"]


# ---------------------------------------------------------------------------------------------------- activations
def geglu_case(K, dev, M, C, seed=0):
    """GEGLU (pack_geglu packing, 128-column granules) on integer pre-activations with value and gate spread over about
    -3 .. 3 (density sqrt(4 / C): about 4 non-zero products per output) + half-integer fp16 bias."""
    p = math.sqrt(4.0 / C)
    A = ternary((M, C), seed, p).to(dev)
    Wt = ternary((8 * C, C), seed + 1, p).to(dev)
    bh = halves((8 * C,), seed + 2, 1.0).half().to(dev)
    wp, bp = K.pack_geglu(Wt, bh)
    out = K.gemm(A, wp, bias=bp, mode=GEGLU)
    h = A.double() @ Wt.double().t() + bh.double()
    v, g = h[:, :4 * C], h[:, 4 * C:]
    assert float(g.min()) <= -3 and float(g.max()) >= 3, "probe premise: gates spread over -3 .. 3"
    y, bound = geglu_bound(v, g)
    return NP.compare(out, y, bound, f"GEGLU M {M} C {C}")


def qgelu_case(K, dev, M, bn, Kd=768, N=3072, seed=0):
    """quick-GELU (CLIP's fc1 shape) on integer pre-activations + half-integer bias."""
    p = math.sqrt(4.0 / Kd)
    A = ternary((M, Kd), seed, p).to(dev)
    Wt = ternary((N, Kd), seed + 1, p).to(dev)
    b = halves((N,), seed + 2).to(dev)
    out = K.gemm(A, Wt, bias=b, bn=bn, mode=QGELU)
    v = A.double() @ Wt.double().t() + b.double()
    r = CP.compare_qgelu(out.cpu(), v.cpu())
    r["what"] = f"quick-GELU M {M} bn {bn}"
    return r
