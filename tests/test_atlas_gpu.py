"""Point-drag propagation on the GPU: vs_imlp_forward per element against fp64 within a bound derived from K fp32 FMAs
per layer, vs_atlas_propagate against the reference fixture (tests/golden/atlas.pt: every track and visibility decision
exact), its launch count, and the descriptors it must reject before any launch."""
import ctypes as C
import json
import math
import os

import pytest
import torch

from oracle import make_golden_atlas as M
from videoswap_b200 import _lib, atlas

pytestmark = pytest.mark.gpu

GOLD = torch.load(os.path.join(os.path.dirname(__file__), "golden", "atlas.pt"), weights_only=False)
U = 2.0 ** -24
CFGS = (M.FG, M.FG_INV, M.ALPHA)


def _net(cfg, sd):
    n = atlas.IMLP_Hash(**cfg, device="cuda")
    n.load_state_dict(sd)
    return n


def imlp64(sd, cfg, x32):
    """(fp64 output, per-element bound on an fp32 evaluation's error).  The encoding's arguments x b_j are rounded to
    fp32 as the kernel does; sinf / cosf / tanhf are within 2 ulp; a K-term fp32 dot product plus bias is within
    (K + 1) u (|W| |x| + |b|), and an input error e propagates as |W| e."""
    x32 = x32.float().cpu()
    if cfg["pe_type"] == "encoding":
        b = torch.tensor([(2 ** j) * math.pi for j in range(cfg["pe_dim"])], dtype=torch.float32)
        proj = (x32[:, :, None] * b).double()
        h = torch.cat((torch.sin(proj), torch.cos(proj)), 1).transpose(2, 1).reshape(x32.shape[0], -1)
        e = torch.full_like(h, 2 * U)
    else:
        h, e = x32.double(), torch.zeros(x32.shape, dtype=torch.float64)
    inp, e_inp = h, e
    for i in range(cfg["mlp_layers"]):
        if i > 0:
            h = h.clamp_min(0)
        if i in cfg["skip_layers"]:
            h, e = torch.cat((h, inp), 1), torch.cat((e, e_inp), 1)
        W, bias = sd[f"hidden.{i}.weight"].double(), sd[f"hidden.{i}.bias"].double()
        K = W.shape[1]
        e = e @ W.abs().t() + (K + 1) * U * 1.01 * (h.abs() @ W.abs().t() + bias.abs())
        h = h @ W.t() + bias
    if cfg.get("use_tanh", True):
        h, e = torch.tanh(h), e + 2 * U
    return h, e


@pytest.mark.parametrize("rows", [1, 63, 65, 3000])
@pytest.mark.parametrize("case", ["fg", "fg_inverse", "alpha", "skip", "width128"])
def test_imlp_forward_against_fp64(case, rows):
    cfg = {"fg": M.FG, "fg_inverse": M.FG_INV, "alpha": M.ALPHA, "skip": M.NETWORK,
           "width128": dict(M.NETWORK, hidden_dim=128, mlp_layers=5, skip_layers=[2])}[case]
    sd = M.seeded_imlp(cfg, 100 + rows, 1.5)
    x = torch.rand((rows, cfg["input_dim"]), generator=torch.Generator().manual_seed(rows)) * 2 - 1
    got = _net(cfg, sd)(x.cuda())
    torch.cuda.synchronize()
    ref, bound = imlp64(sd, cfg, x)
    err = (got.double().cpu() - ref).abs()
    assert torch.isfinite(got).all()
    assert (err <= bound).all(), (case, rows, float((err / bound).max()))
    # the worst-case bound grows with sum |W| per layer and is loose for deep networks; a wrong weight, layout or
    # activation moves outputs by O(0.1), so also hold the observed error to fp32 reordering size
    assert float(err.max()) < 1e-4, (case, rows, float(err.max()))


def test_network_case_matches_reference():
    sd = M.seeded_imlp(M.NETWORK, GOLD["network"]["seed"])
    got = _net(M.NETWORK, sd)(M.network_input().cuda()).cpu().double()
    ref, bound = imlp64(sd, M.NETWORK, M.network_input())
    assert ((got - GOLD["network"]["out"].double()).abs() <= 2 * bound).all()


def _nets(nets_sd):
    return tuple(_net(c, sd) for c, sd in zip(CFGS, nets_sd))


def _files(tmp_path):
    src = tmp_path / f"{GOLD['keyframe']:05d}.json"
    tgt = tmp_path / "edit.json"
    src.write_text(json.dumps(GOLD["source"]))
    tgt.write_text(json.dumps(GOLD["target"]))
    return str(src), str(tgt)


@pytest.mark.parametrize("case", ["main", "tie", "threshold"])
def test_propagation_tracks_exact(tmp_path, case):
    sds = M.nets_for(GOLD["seed"])
    sds, ld, want = {"main": (sds, GOLD["larger_dim"], GOLD["pred_tracks"]),
                     "tie": (M.tie_nets(sds), GOLD["tie"]["larger_dim"], GOLD["tie"]["pred_tracks"]),
                     "threshold": (M.threshold_nets(sds), GOLD["larger_dim"], GOLD["threshold"]["pred_tracks"])}[case]
    src, tgt = _files(tmp_path)
    out = atlas.propagate_point_sequence(src, M.source_tap(), tgt, *_nets(sds), larger_dim=ld,
                                         number_of_frames=GOLD["F"])
    assert out["pred_tracks"].device.type == "cpu" and out["pred_tracks"].dtype == torch.float32
    assert torch.equal(out["pred_tracks"], want)


def test_propagation_stages_against_fixture():
    """Normalised inputs and the frame axis bit-exact; each network's outputs within the fp32 bound of an fp64 evaluation
    on the kernel's own inputs, and within twice the bound of the fixture's; visibility decisions exact."""
    sds = M.nets_for(GOLD["seed"])
    nets = _nets(sds)
    g = GOLD["stages"]
    P, F = 4, GOLD["F"]
    from tests import atlas_oracle as A
    cols, pts, t_key = A.normalised_points(GOLD["source"], GOLD["target"], M.source_tap()["point_name2id"],
                                           GOLD["keyframe"], GOLD["larger_dim"], F)
    res, ws = atlas.propagate_points(nets, pts, float(t_key), F, GOLD["larger_dim"])
    st = {k: v.cpu() for k, v in atlas.stages(ws, P, F).items()}
    assert torch.equal(st["fg_in"], g["fg_in"])
    assert torch.equal(st["inv_in"][:, 2], g["inv_in"][:, 2])
    for name, (cfg, sd), rows_in, rows_out in (("fg", (M.FG, sds[0]), "fg_in", "fg_out"),
                                               ("inv", (M.FG_INV, sds[1]), "inv_in", "inv_out")):
        ref, bound = imlp64(sd, cfg, st[rows_in])
        assert ((st[rows_out].double() - ref).abs() <= bound).all(), name
    assert ((st["fg_out"].double() - g["fg_out"].double()).abs() <= 2 * imlp64(sds[0], M.FG, g["fg_in"])[1]).all()
    ref, bound = imlp64(sds[2], M.ALPHA, st["inv_out"][:P * F])
    assert ((st["alpha"].double() - ref[:, 0]).abs() <= bound[:, 0]).all()
    assert ((st["alpha"] - g["alpha"]).abs() <= 2e-4).all()
    # the finalize arithmetic on the kernel's own stages, and the result against the fixture
    b, xu, xv = st["inv_out"].view(3, P * F, 3)
    J = torch.stack([(xu - b) / 0.1, (xv - b) / 0.05], 1)[..., :2]
    assert torch.allclose(st["J_inv"], J, rtol=1e-6, atol=1e-6)
    assert torch.allclose(st["J_inv"], g["J_inv"], atol=1e-4) and torch.allclose(st["J_fg"], g["J_fg"], atol=1e-4)
    assert torch.allclose(st["warp"], g["warp"], atol=1e-5)
    vis = 0.5 * (st["alpha"] + 1.0) > 0.5
    assert torch.equal(vis, 0.5 * (g["alpha"] + 1.0) > 0.5)
    assert torch.equal(res.cpu(), GOLD["pred_tracks"][:, cols])


def test_launch_count_does_not_depend_on_points_or_frames():
    nets = _nets(M.nets_for(GOLD["seed"]))
    counts = []
    for P, F in ((1, 16), (6, 72)):
        pts = torch.rand((P, 4), generator=torch.Generator().manual_seed(P)) * 0.2
        n0 = _lib.lib().vs_launch_count()
        atlas.propagate_points(nets, pts, -0.5, F, 768)
        counts.append(_lib.lib().vs_launch_count() - n0)
    torch.cuda.synchronize()
    assert counts[0] == counts[1] == 6, counts


def test_malformed_descriptors_are_rejected_before_any_launch():
    nets = _nets(M.nets_for(GOLD["seed"]))
    x = torch.zeros((4, 3), device="cuda")
    out = torch.zeros((4, 3), device="cuda")
    pts = torch.zeros((2, 4), device="cuda")
    ws = torch.zeros((21 * 2 + 25 * 2 * 8,), device="cuda")
    tr = torch.zeros((8, 2, 2), device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    L = _lib.lib()

    def bad(**kw):
        d = nets[1].desc()
        for k, v in kw.items():
            setattr(d, k, v)
        return d

    cases = [bad(hidden_dim=48), bad(hidden_dim=512), bad(mlp_layers=0), bad(skip_mask=1), bad(skip_mask=1 << 6),
             bad(output_dim=0), bad(pe_dim=-1), bad(params=None)]
    n0 = L.vs_launch_count()
    for d in cases:
        assert L.vs_imlp_forward(s, C.byref(d), C.c_void_p(x.data_ptr()), 4, C.c_void_p(out.data_ptr())) != 0
    d = nets[1].desc()
    assert L.vs_imlp_forward(s, C.byref(d), C.c_void_p(x.data_ptr()), 0, C.c_void_p(out.data_ptr())) != 0
    descs = [n.desc() for n in nets]

    def prop(P, F, ds=descs):
        return L.vs_atlas_propagate(s, *[C.byref(d) for d in ds], C.c_void_p(pts.data_ptr()), -0.5, P, F, 768,
                                    C.c_void_p(ws.data_ptr()), C.c_void_p(tr.data_ptr()))

    assert prop(0, 8) != 0 and prop(2, 0) != 0
    assert prop(2, 8, [descs[1], descs[1], descs[2]]) != 0          # FG must map 3 -> 2
    assert prop(2, 8, [descs[0], bad(mlp_layers=0), descs[2]]) != 0
    assert L.vs_launch_count() == n0
    assert prop(2, 8) == 0 and L.vs_launch_count() == n0 + 6
    torch.cuda.synchronize()
