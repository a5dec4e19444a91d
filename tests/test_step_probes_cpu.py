"""The power of the step probes (tests/step_probes.py), shown without a GPU.  A torch emulation of the kernels'
arithmetic -- small_linear's lane-strided fp32 pair sums and butterfly reduction, adapter_splat's per-cell fp32 gather
of r16(feat) * wsum with the r16 coordinate roundings, the fp32 sinusoid -- passes every comparator (the exact ones
exactly, the bounded ones with 2x margin), and every planted bug fails.  The fp64 restatement reproduces the two
adapter fixtures the reference's own SparsePointAdapter wrote, and the bugs the existing adapter-golden bounds and
scalar-timestep UNet tests let through are recorded."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import step_probes as S
from videoswap_b200.spec import UNetConfig, adapter_param_shapes, unet_param_shapes
from videoswap_b200.weights import seeded_state_dict

GOLD = os.path.join(os.path.dirname(__file__), "golden")
U32 = 2.0 ** -24


# ------------------------------------------------------------------------------------------------------ emulation
def _silu32(x):
    return x / (1 + torch.exp(-x))


def small_linear(x, W, b, silu_in, silu_out, mutation=None):
    """small_linear_kernel: lane l of output n sums (a w_k + b w_k+1) over k = 2 l + 64 i in fp32, the 32 lanes meet in
    a shfl_xor butterfly, then the bias (and SiLU) in fp32."""
    x, W = x.float(), W.float()
    R, K = x.shape
    N = W.shape[0]
    Kp = -(-K // 64) * 64
    xs = torch.zeros(R, Kp)
    xs[:, :K] = _silu32(x) if silu_in else x
    Ws = torch.zeros(N, Kp)
    Ws[:, :K] = W
    if mutation == "k_tail" and K % 64:
        xs[:, K - 2:K] = 0                                       # the lane loop stops before the last partial pair
    if mutation == "row0":
        xs = xs[:1].expand(R, Kp)                                # every row reads row 0
    xs, Ws = xs.view(R, Kp // 64, 32, 2), Ws.view(N, Kp // 64, 32, 2)
    acc = torch.zeros(R, N, 32)
    for i in range(Kp // 64):
        a, w = xs[:, i], Ws[:, i]
        acc = acc + (a[:, None, :, 0] * w[None, :, :, 0] + a[:, None, :, 1] * w[None, :, :, 1])
    lanes = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        acc = acc + acc[..., lanes ^ o]
    v = acc[..., 0] + b.float()
    if silu_out:
        v = _silu32(v)
    if mutation == "rows_ge8":
        v[8:] = 0                                                # the row loop never leaves its first block
    return v


def _f32(v):
    return np.float32(v)


def emulate_splat(feat, tracks, mask, F_, P, C, h, w, rate, c16, scale, mutation=None):
    """adapter_splat_kernel: every cell gathers, point by point, r16(feat) * wsum in fp32, wsum being the cell's fp32 sum
    of the point's weights in corner order; then fp16(r16(acc) * scale)."""
    def r16(v, on=c16):
        return _f32(np.float16(v)) if on else _f32(v)

    acc = torch.zeros(F_, h, w, C)
    feat16 = feat.half().float() if c16 else feat.float()
    tr = tracks.reshape(-1, 2).numpy()
    for pt in range(P):
        if mask is not None and not int(mask[pt]) and mutation != "mask_ignored":
            continue
        for f in range(F_):
            row = pt * F_ + f if mutation == "pt_f_swap" else f * P + pt
            ix, iy = (1, 0) if mutation == "xy_swap" else (0, 1)
            px, py = r16(tr[row, ix]), r16(tr[row, iy])
            if (px <= 0 or py <= 0) if mutation == "le0" else (px < 0 or py < 0):
                continue
            fx, fy = r16(px / _f32(rate)), r16(py / _f32(rate))
            x1, y1 = int(fx), int(fy)
            xf = r16(fx - _f32(x1), c16 and mutation != "xf_unrounded")
            yf = r16(fy - _f32(y1))
            x2, y2 = x1 + 1, y1 + 1
            x1, x2 = max(min(x1, w - 1), 0), max(min(x2, (h if mutation == "x2_clamp_h" else w) - 1), 0)
            y1, y2 = max(min(y1, h - 1), 0), max(min(y2, h - 1), 0)
            wr = c16 and mutation != "weights_unrounded"
            ox, oy = r16(1 - xf, wr), r16(1 - yf)
            corners = [(y1, x1, r16(ox * oy, wr)), (y1, x1 if mutation == "x2_on_x1" else x2, r16(xf * oy, wr)),
                       (y2, x1, r16(ox * yf, wr)), (y2, x2, r16(xf * yf, wr))]
            cells = {}
            for cy, cx, wt in corners:
                if 0 <= cx < w:
                    cells[(cy, cx)] = _f32(cells.get((cy, cx), _f32(0)) + wt)
            for (cy, cx), ws in cells.items():
                if ws != 0:
                    acc[f, cy, cx] += feat16[pt] * float(ws)
    return (acc.half().float() * scale).half() if c16 else (acc * scale).half()


def emulate_adapter(mutation=None):
    def run(w0, b0, w1, b1, pe, tracks, h, w, rate, mask, coord_fp16, scale):
        hid = small_linear(pe, w0, b0.float(), False, True, mutation)
        feat = small_linear(hid, w1, b1.float(), False, False, mutation)
        F_, P = tracks.shape[:2]
        return emulate_splat(feat, tracks, mask, F_, P, w1.shape[0], h, w, rate, bool(coord_fp16), scale, mutation)
    return run


CFG = UNetConfig()
_SD = {}


def time_sd():
    """The time-embedding weights of the SD-1.5 shapes, seeded, as fp32 holding fp16 values."""
    if "sd" not in _SD:
        shapes = unet_param_shapes(CFG)
        _SD["sd"] = {k: v.half().float() for k, v in seeded_state_dict({k: shapes[k] for k in S.time_param_names(CFG)}, seed=0).items()}
    return _SD["sd"]


def emulate_time(mutation=None):
    sd = time_sd()
    layout = S.tproj_layout(CFG)
    wp = torch.cat([sd[f"{n}.time_emb_proj.weight"] for n, _, _ in layout])
    bp = torch.cat([sd[f"{n}.time_emb_proj.bias"] for n, _, _ in layout])

    def run(t):
        half = CFG.block_out_channels[0] // 2
        freq = torch.exp(-9.210340371976184 * torch.arange(half, dtype=torch.float32) / half)
        arg = t.float()[:, None] * freq[None, :]
        c, s = torch.cos(arg), torch.sin(arg)
        te0 = torch.cat([s, c] if mutation == "sincos" else [c, s], -1)
        te1 = small_linear(te0, sd["time_embedding.linear_1.weight"], sd["time_embedding.linear_1.bias"], False, True)
        emb = small_linear(te1, sd["time_embedding.linear_2.weight"], sd["time_embedding.linear_2.bias"], False, False)
        return emb, small_linear(emb, wp, bp, True, False, mutation)
    return run


# ------------------------------------------------------------------------------------------------------- cases
def _cells(level, P, kind="regimes", **kw):
    return lambda fn: S.check_adapter_cells(fn, level, P, kind, dev="cpu", **kw)


def _geom(name, level, c16, scale=1.0):
    return lambda fn: S.check_adapter_geometry(fn, name, level, c16, scale, dev="cpu")


def _quant(level, c16, axis=0, scale=1.0):
    return lambda fn: S.check_adapter_quant(fn, level, c16, axis, scale, dev="cpu")


T9 = [0, 1, 500, 981, 999, 21, 261, 741, 2]
ADAPTER_CASES = {
    "cells_L0_regimes_P9": _cells(0, 9),
    "cells_L3_regimes_P9_fp32coords": _cells(3, 9, coord_fp16=False),
    "dense_L1_P9": _cells(1, 9, "dense"),
    "dense_L0_P33_tail_1278_98": _cells(0, 33, "dense", E=1278, mid=98),
    "edges_L3": _geom("edges", 3, True),
    "edges_L0_fp32_scale3": _geom("edges", 0, False, 3.0),
    "signs_L1_fp16": _geom("signs", 1, True),
    "signs_L1_fp32": _geom("signs", 1, False),
    "mask_L2": _geom("mask", 2, True, 0.5),
    "frames_L0": _geom("frames", 0, True),
    "pile_L2": _geom("pile", 2, False, 3.0),
    "floor_L3": _geom("floor", 3, True),
    "one_cell_L3": _geom("one_cell", 3, False),
    "quant_L0_fp16": _quant(0, True),
    "quant_L3_fp16_tall": _quant(3, True, 1, 3.0),
    "quant_L1_fp32": _quant(1, False),
}
BOUNDED = {"quant_L0_fp16", "quant_L3_fp16_tall", "quant_L1_fp32"}
TIME_CASES = {"time_B1": lambda fn: S.check_time_embedding(fn, time_sd(), CFG, [999], dev="cpu"),
              "time_B2": lambda fn: S.check_time_embedding(fn, time_sd(), CFG, [981, 1], dev="cpu"),
              "time_B9": lambda fn: S.check_time_embedding(fn, time_sd(), CFG, T9, dev="cpu")}

# (emulation, case that must reject it)
MUTATIONS = {
    "x_and_y_swapped": (lambda: emulate_adapter("xy_swap"), ADAPTER_CASES["frames_L0"]),
    "x2_clamped_with_h": (lambda: emulate_adapter("x2_clamp_h"), ADAPTER_CASES["floor_L3"]),
    "x2_weight_on_x1": (lambda: emulate_adapter("x2_on_x1"), ADAPTER_CASES["edges_L3"]),
    "mask_ignored": (lambda: emulate_adapter("mask_ignored"), ADAPTER_CASES["mask_L2"]),
    "point_frame_index_swapped": (lambda: emulate_adapter("pt_f_swap"), ADAPTER_CASES["frames_L0"]),
    "weights_not_rounded_to_fp16": (lambda: emulate_adapter("weights_unrounded"), ADAPTER_CASES["quant_L3_fp16_tall"]),
    "lt0_made_le0": (lambda: emulate_adapter("le0"), ADAPTER_CASES["signs_L1_fp16"]),
    "last_k_pair_dropped": (lambda: emulate_adapter("k_tail"), ADAPTER_CASES["dense_L0_P33_tail_1278_98"]),
    "rows_from_8_skipped": (lambda: emulate_adapter("rows_ge8"), ADAPTER_CASES["cells_L0_regimes_P9"]),
    "sin_and_cos_swapped": (lambda: emulate_time("sincos"), TIME_CASES["time_B1"]),
    "every_row_reads_row_0": (lambda: emulate_time("row0"), TIME_CASES["time_B2"]),
}


def _msg(name, r):
    return f"{name}: {r['what']} (err {r['err']:.3g})"


@pytest.mark.parametrize("name", sorted(ADAPTER_CASES))
def test_emulated_adapter_passes(name):
    r = ADAPTER_CASES[name](emulate_adapter())
    assert r["ok"], _msg(name, r)
    if name in BOUNDED:
        assert r["err"] <= 0.5, _msg(name, r)
    else:
        assert r["err"] == 0, _msg(name, r)


@pytest.mark.parametrize("name", sorted(TIME_CASES))
def test_emulated_time_embedding_passes_with_margin(name):
    r = TIME_CASES[name](emulate_time())
    assert r["ok"] and r["err"] <= 0.5, _msg(name, r)


@pytest.mark.parametrize("name", sorted(MUTATIONS))
def test_planted_mutation_is_rejected(name):
    emu, case = MUTATIONS[name]
    r = case(emu())
    assert not r["ok"], _msg(name, r)


def test_xf_rounding_cannot_change_anything():
    """r16(fx - x1) in adapter_splat is an identity: for every non-negative fp16 fx, fx minus its integer part keeps fx's
    ulp and needs fewer bits, so it is an fp16 value.  Dropping that r16 is not a bug any probe could see; dropping the
    roundings of the weights formed from it is (weights_not_rounded_to_fp16)."""
    fx = torch.arange(0, 0x7C00, dtype=torch.int32).to(torch.int16).view(torch.float16).double()   # all finite fp16 >= 0
    frac = fx - torch.trunc(fx)
    assert torch.equal(frac.half().double(), frac)
    r = ADAPTER_CASES["quant_L0_fp16"](emulate_adapter("xf_unrounded"))
    assert r["ok"] and r["err"] <= 0.5, _msg("xf_unrounded", r)


# ------------------------------------------------------------------------------------- the reference's fixtures
def _golden_inputs(fp16):
    from oracle.make_golden import adapter_fp16_inputs, densify
    sd = seeded_state_dict(adapter_param_shapes(), seed=5)
    if fp16:
        g = torch.load(os.path.join(GOLD, "adapter_fp16.pt"))
        tracks, emb, size, index_list = adapter_fp16_inputs()
    else:
        g = torch.load(os.path.join(GOLD, "adapter.pt"))
        tracks, emb, size, index_list = g["tracks"], g["emb"], g["size"], None
    return sd, tracks, emb, size, index_list, densify(g["maps_sparse"])


@pytest.mark.parametrize("fp16", [True, False])
def test_restatement_reproduces_reference_fixtures(fp16):
    """splat_ref on the reference's own MLP output matches adapter.pt (fp32) / adapter_fp16.pt (weights, coordinates
    and maps in fp16) with the same support, within the reference's own rounding: fp16, each product feat w and each
    += rounds (2 n 2^-11 A); fp32, the same with u plus the two fp32 MLPs' dot-product error carried through the
    weights."""
    sd, tracks, emb, size, index_list, ref = _golden_inputs(fp16)
    u = 2.0 ** -11 if fp16 else 2.0 ** -24
    dt = torch.float16 if fp16 else torch.float32
    mask = None if index_list is None else torch.tensor([int(i in index_list) for i in range(tracks.shape[1])])
    for lv, (C, rate) in enumerate(S.LEVELS):
        w0, b0, w1, b1 = (sd[f"model_list.{lv}.mlp.{i}.{s}"].to(dt) for i in (0, 2) for s in ("weight", "bias"))
        x = emb.to(dt)
        feat = F.linear(F.silu(F.linear(x, w0, b0)), w1, b1).double()
        # the fixture's MLP ran on another machine: fp32 dot products in some order, each layer rounded to `dt`
        W0, W1 = w0.double().abs(), w1.double().abs()
        hd = F.linear(x.double(), w0.double(), b0.double())
        sd_ = F.silu(hd)
        dh = 2 * (W0.shape[1] + 1) * U32 * (x.double().abs() @ W0.t() + b0.double().abs()) + 2 * u * hd.abs()
        ds = 1.1 * dh + 2 * u * sd_.abs()
        dfeat = ds @ W1.t() + 2 * (W1.shape[1] + 1) * U32 * (sd_.abs() @ W1.t() + b1.double().abs()) + 2 * u * feat.abs()
        h, w = size[1] // rate, size[0] // rate
        m, A, n = S.splat_ref(feat, tracks, h, w, rate, mask, coord_fp16=fp16)
        dm = S.splat_ref(dfeat, tracks, h, w, rate, mask, coord_fp16=fp16)[0]
        bound = 2 * n * u * A * (1 + 2.0 ** -10) + dm + 2 * n * 2.0 ** -25
        r = ref[lv].double().permute(0, 2, 3, 1)
        assert torch.equal((m != 0).any(-1), (r != 0).any(-1)), lv
        ratio = ((m - r).abs() / bound.clamp_min(1e-300)).max().item()
        assert ratio <= 1.0, (lv, ratio)


# ------------------------------------------------------------------------------------- what the old tests saw
def _old_adapter_golden(mutation):
    """The existing adapter tests of tests/test_unet_gpu.py on the emulation: adapter.pt with fp32 coordinates,
    max|d| <= 2^-8 max|ref| + 2e-3, and adapter_fp16.pt with fp16 coordinates and the index list, max|d| <= 2^-7 max|ref|
    + 4e-3 with the same support.  True when the mutated emulation passes both."""
    emu = emulate_adapter(mutation)
    for fp16 in (False, True):
        sd, tracks, emb, size, index_list, ref = _golden_inputs(fp16)
        mask = None if index_list is None else torch.tensor([int(i in index_list) for i in range(tracks.shape[1])])
        for lv, (C, rate) in enumerate(S.LEVELS):
            w0, b0, w1, b1 = (sd[f"model_list.{lv}.mlp.{i}.{s}"].half() for i in (0, 2) for s in ("weight", "bias"))
            h, w = size[1] // rate, size[0] // rate
            out = emu(w0, b0, w1, b1, emb.float(), tracks.float(), h, w, rate, mask, fp16, 1.0).float()
            r = ref[lv].float().permute(0, 2, 3, 1)
            tol = (2 ** -7 * r.abs().max() + 4e-3) if fp16 else (2 ** -8 * r.abs().max() + 2e-3)
            if (out - r).abs().max() > tol:
                return False
            if fp16 and not torch.equal((out != 0).any(-1), (r != 0).any(-1)):
                return False
    return True


ADAPTER_BLIND = ["weights_unrounded", "rows_ge8"]
ADAPTER_CAUGHT = ["xy_swap", "x2_on_x1", "mask_ignored", "pt_f_swap"]


@pytest.mark.parametrize("mutation", ADAPTER_BLIND)
def test_adapter_golden_bound_passes_the_bug(mutation):
    assert _old_adapter_golden(mutation), f"{mutation}: the adapter-golden bound caught it after all"


@pytest.mark.parametrize("mutation", ADAPTER_CAUGHT)
def test_adapter_golden_bound_rejects_the_bug(mutation):
    assert not _old_adapter_golden(mutation), f"{mutation}: the adapter-golden bound let it through"


def test_scalar_timestep_cannot_see_a_row_mix_up():
    """Every UNet test passes one scalar timestep, so all B rows of the projections are equal and a row mix-up gives
    bit-identical rows; the per-row probe with distinct timesteps rejects it (every_row_reads_row_0)."""
    t = torch.tensor([981.0, 981.0])
    e, p = emulate_time()(t)
    e2, p2 = emulate_time("row0")(t)
    assert torch.equal(e, e2) and torch.equal(p, p2)
