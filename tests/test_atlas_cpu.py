"""Point-drag propagation on the CPU: the torch restatement (tests/atlas_oracle.py) against the reference fixture
(oracle/make_golden_atlas.py -> tests/golden/atlas.pt), the planted bugs that must break it, and the host logic of
videoswap_b200.atlas with the native propagation replaced by the restatement."""
import json
import os

import pytest
import torch

from oracle import make_golden_atlas as M
from tests import atlas_oracle as A
from videoswap_b200 import atlas, formats

GOLD = torch.load(os.path.join(os.path.dirname(__file__), "golden", "atlas.pt"), weights_only=False)
CFGS = (M.FG, M.FG_INV, M.ALPHA)


def _nets():
    return M.nets_for(GOLD["seed"])


def _run(nets=None, larger_dim=None):
    return A.propagate_tap(nets or _nets(), CFGS, GOLD["source"], M.source_tap(), GOLD["target"], GOLD["keyframe"],
                           larger_dim or GOLD["larger_dim"], GOLD["F"])


def _close(a, b, atol=2e-6, rtol=1e-5):
    return torch.allclose(a, b, atol=atol, rtol=rtol)


def _matches():
    out, st = _run()
    g = GOLD["stages"]
    ok = torch.equal(out["pred_tracks"], GOLD["pred_tracks"])
    ok &= torch.equal(st["fg_in"], g["fg_in"]) and torch.equal(st["inv_in"][:, 2], g["inv_in"][:, 2])
    ok &= _close(st["alpha"], g["alpha"], atol=2e-4)
    tie, _ = _run(M.tie_nets(_nets()), GOLD["tie"]["larger_dim"])
    ok &= torch.equal(tie["pred_tracks"], GOLD["tie"]["pred_tracks"])
    thr, _ = _run(M.threshold_nets(_nets()))
    ok &= torch.equal(thr["pred_tracks"], GOLD["threshold"]["pred_tracks"])
    net = A.imlp(M.seeded_imlp(M.NETWORK, GOLD["network"]["seed"]), M.NETWORK, M.network_input())
    ok &= _close(net, GOLD["network"]["out"])
    return bool(ok)


def test_restatement_reproduces_every_stage():
    """Normalised inputs and the frame axis bit-exact; network outputs, Jacobians, alpha and warps to fp32 reordering;
    every track exact (the fixture's margins: >= 0.01 px from a half-integer, alpha >= 1e-4 from the threshold)."""
    out, st = _run()
    g = GOLD["stages"]
    P, F = st["J_fg"].shape[0], GOLD["F"]
    assert P == 4 and F == 72
    assert torch.equal(st["fg_in"], g["fg_in"])
    assert torch.equal(st["inv_in"][:, 2], g["inv_in"][:, 2])
    # batching reorders fp32 sums in the last bits; the finite differences scale that by 10-20, and F_Alpha (frequencies
    # up to 16 pi) by about 100
    for k, tol in (("fg_out", 2e-6), ("J_fg", 5e-5), ("inv_in", 2e-6), ("inv_out", 5e-6), ("J_inv", 5e-5),
                   ("warp", 5e-6), ("alpha", 2e-4)):
        assert _close(st[k], g[k], atol=tol), k
    assert _close(A.imlp(_nets()[2], M.ALPHA, g["alpha_in"])[:, 0], g["alpha"], atol=1e-6)
    assert _close(st["inv_out"][:P * F], g["alpha_in"], atol=5e-6)
    assert torch.equal(out["pred_tracks"], GOLD["pred_tracks"])
    assert out["pred_tracks"].dtype == torch.float32
    # the fixture exercises what it claims to: moved points with visible and occluded frames, untouched columns
    vis = st["visible"]
    assert vis.any(0).all() and (~vis).any(0).all()
    src = M.source_tap()["pred_tracks"]
    for name in ("p2", "p4", "p6"):
        c = M.NAMES.index(name)
        assert torch.equal(out["pred_tracks"][:, c], src[:, c])
    motion = (st["warp"].view(P, F, 2).amax(1) - st["warp"].view(P, F, 2).amin(1)) * GOLD["larger_dim"] / 2
    assert (motion.amax(1) >= 20).all()


def test_tie_case_rounds_half_to_even():
    tie, st = _run(M.tie_nets(_nets()), GOLD["tie"]["larger_dim"])
    assert torch.equal(tie["pred_tracks"], GOLD["tie"]["pred_tracks"])
    vis = st["visible"]
    assert vis.any() and (~vis).any() and (st["tracks"][vis] == 382).all()


def test_threshold_case_is_not_visible():
    thr, st = _run(M.threshold_nets(_nets()))
    assert torch.equal(thr["pred_tracks"], GOLD["threshold"]["pred_tracks"])
    assert (st["alpha"] == 0).all() and not st["visible"].any()


def test_network_case_with_skip_layers():
    net = A.imlp(M.seeded_imlp(M.NETWORK, GOLD["network"]["seed"]), M.NETWORK, M.network_input())
    assert _close(net, GOLD["network"]["out"])


def _bug_swap_xy(v):
    return v[0], v[1]


def _bug_alpha_at_frame_t(xyt_pred, t):
    return torch.cat([xyt_pred[:, :2], t], 1)


def _bug_ge(alpha):
    return 0.5 * (alpha + 1.0) >= 0.5


def _bug_half_up(w, larger_dim):
    return torch.floor((w + 1) / 2 * larger_dim + 0.5)


def _bug_no_clear(tracks, col):
    pass


def _bug_pe_transposed(x, pe_dim):
    b = torch.tensor([(2 ** j) * 3.141592653589793 for j in range(pe_dim)], dtype=x.dtype)
    proj = x[:, :, None] * b
    return torch.cat((torch.sin(proj), torch.cos(proj)), 1).reshape(x.shape[0], -1)


@pytest.mark.parametrize("name,fn", [("point_xy", _bug_swap_xy), ("alpha_input", _bug_alpha_at_frame_t),
                                     ("visible", _bug_ge), ("to_pixel", _bug_half_up),
                                     ("clear_column", _bug_no_clear), ("encode", _bug_pe_transposed)])
def test_planted_bugs_are_caught(monkeypatch, name, fn):
    assert _matches()
    monkeypatch.setattr(A, name, fn)
    assert not _matches(), name


# ------------------------------------------------------------------------------------------------------------ host logic
def test_atlas_dims_needs_only_frames(tmp_path):
    frames = tmp_path / "frames"
    frames.mkdir()
    for i in range(5):
        (frames / f"{i:05d}.jpg").write_bytes(b"")
    opt = {"frame_path": str(frames), "mask_path": str(tmp_path / "none"), "flow_path": str(tmp_path / "none"),
           "res_x": 768, "res_y": 448, "max_frames": 72}
    assert atlas.atlas_dims(opt) == (5, 768)
    assert atlas.atlas_dims(dict(opt, max_frames=3, res_x=256, res_y=512)) == (3, 512)


@pytest.mark.parametrize("kw", [dict(pe_type="hash_encoding"), dict(mlp_type="tcnn")])
def test_tinycudann_configs_are_rejected(kw):
    with pytest.raises(NotImplementedError, match="tinycudann"):
        atlas.IMLP_Hash(**dict(dict(M.FG), **kw), device="cpu")


def test_strict_checkpoint_loading():
    net = atlas.IMLP_Hash(**M.ALPHA, device="cpu")
    sd = M.seeded_imlp(M.ALPHA, 1)
    net.load_state_dict(sd)
    assert torch.equal(net.params["hidden.3.weight"], sd["hidden.3.weight"])
    with pytest.raises(KeyError):
        net.load_state_dict({k: v for k, v in sd.items() if k != "hidden.7.bias"})
    with pytest.raises(KeyError):
        net.load_state_dict(dict(sd, extra=torch.zeros(1)))
    with pytest.raises(ValueError):
        net.load_state_dict(dict(sd, **{"hidden.0.weight": torch.zeros(256, 31)}))
    with pytest.raises(ValueError):
        atlas.IMLP_Hash(**dict(M.NETWORK, skip_layers=[8]), device="cpu")


def test_packed_parameters_follow_the_header_layout():
    net = atlas.IMLP_Hash(**M.NETWORK, device="cpu")
    sd = M.seeded_imlp(M.NETWORK, 3)
    net.load_state_dict(sd)
    o = 0
    for i, (n, k) in enumerate(M.layer_shapes(M.NETWORK)):
        assert torch.equal(net.packed[o:o + k * n].view(k, n), sd[f"hidden.{i}.weight"].t())
        o += k * n
        assert torch.equal(net.packed[o:o + n], sd[f"hidden.{i}.bias"])
        o += n
    assert o == net.packed.numel()
    d = net.desc()
    assert (d.input_dim, d.output_dim, d.pe_dim, d.skip_mask, d.mlp_layers) == (2, 3, 10, (1 << 4) | (1 << 7), 8)


def _fake_native(nets, pts, t_key, F, larger_dim):
    """vs_atlas_propagate's contract computed by the restatement on the CPU."""
    st = A.propagate(tuple(n.params for n in nets), CFGS, pts, torch.tensor(t_key, dtype=torch.float32), F, larger_dim)
    return st["tracks"], None


def test_propagate_point_sequence_from_files(tmp_path, monkeypatch):
    """The keyframe comes from the source file's name; files and loaded dicts are accepted; the result loads with
    formats.load_tap; the input TAP is not modified."""
    monkeypatch.setattr(atlas, "propagate_points", _fake_native)
    nets = []
    for cfg, sd in zip(CFGS, _nets()):
        n = atlas.IMLP_Hash(**cfg, device="cpu")
        n.load_state_dict(sd)
        nets.append(n)
    src = tmp_path / f"{GOLD['keyframe']:05d}.json"
    tgt = tmp_path / "edit.json"
    src.write_text(json.dumps(GOLD["source"]))
    tgt.write_text(json.dumps(GOLD["target"]))
    tap = M.source_tap()
    before = tap["pred_tracks"].clone()
    out = atlas.propagate_point_sequence(str(src), tap, str(tgt), *nets, larger_dim=GOLD["larger_dim"],
                                         number_of_frames=GOLD["F"])
    assert torch.equal(out["pred_tracks"], GOLD["pred_tracks"])
    assert torch.equal(tap["pred_tracks"], before)
    torch.save(tap, tmp_path / "TAP.pth")
    out2 = atlas.propagate_point_sequence(GOLD["source"], str(tmp_path / "TAP.pth"), GOLD["target"], *nets,
                                          larger_dim=GOLD["larger_dim"], number_of_frames=GOLD["F"],
                                          keyframe=GOLD["keyframe"])
    assert torch.equal(out2["pred_tracks"], GOLD["pred_tracks"])
    wrong = tmp_path / "00003.json"
    wrong.write_text(json.dumps(GOLD["source"]))
    out3 = atlas.propagate_point_sequence(str(wrong), tap, str(tgt), *nets, larger_dim=GOLD["larger_dim"],
                                          number_of_frames=GOLD["F"])
    assert not torch.equal(out3["pred_tracks"], GOLD["pred_tracks"])
    with pytest.raises(ValueError, match="keyframe"):
        atlas.propagate_point_sequence(GOLD["source"], tap, GOLD["target"], *nets, larger_dim=768, number_of_frames=72)
    cond = formats.load_tap(out)
    assert torch.equal(cond["pred_tracks"], GOLD["pred_tracks"]) and cond["point_name2id"] == tap["point_name2id"]
