"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/atlas.pt from the REFERENCE's own code on the CPU:

  * propagation: propagate_point_displacement.propagate_point_sequence with the reference's IMLP_Hash networks in the
    configuration of its atlas configs (FG_UV_Mapping / FG_UV_Mapping_Inverse: pe_type none, 6 layers; F_Alpha: encoding
    with pe_dim 5, 8 layers; all 256 wide, tanh), F = 72 frames, larger_dim = 768, keyframe 17, 4 of 6 source points
    moved (two are absent from the target file; the TAP file has a seventh point the source file does not name).  Every
    network call, compute_Wm and propogate_point is recorded, so the fixture holds the stages: normalised inputs, FG and
    inverse outputs, Jacobians, alpha, pre-round warps and the final tracks.
  * tie: the same points with larger_dim = 765 and the inverse network's x / y outputs zeroed, so every warp is 0 and
    every visible coordinate is 382.5 before rounding (half to even gives 382).
  * threshold: F_Alpha's last layer zeroed, so 0.5 (alpha + 1) is exactly 0.5 and no frame of a moved point is visible.
  * network: IMLP_Hash with F_Atlas's MLP shape (2 -> 3, pe_dim 10, skip_layers [4, 7], 8 layers) on seeded inputs.

Weights come from seeds (seeded_imlp); the seeds are searched from 0 until every moved point has visible and occluded
frames, moves by at least 20 pixels over the clip, every written coordinate is at least 0.01 px from a half-integer before
rounding and every 0.5 (alpha + 1) is at least 1e-4 from 0.5, so a native implementation can be held to every track.
Imports go through throw-away sys.modules stubs for tinycudann, imageio and omegaconf.OmegaConf; the module global
`device` is set to 'cpu'.

Run where the reference tree is checked out:  VIDEOSWAP_REFERENCE=<checkout> python -m oracle.make_golden_atlas
"""
import copy
import json
import math
import os
import sys
import tempfile
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.make_golden import OUT  # noqa: E402
from oracle.ref_loader import REFERENCE_ROOT  # noqa: E402

FG = dict(input_dim=3, output_dim=2, hidden_dim=256, pe_type="none", pe_dim=4, mlp_type="origin", mlp_layers=6,
          skip_layers=[])
FG_INV = dict(FG, output_dim=3)
ALPHA = dict(input_dim=3, output_dim=1, hidden_dim=256, pe_type="encoding", pe_dim=5, mlp_type="origin", mlp_layers=8,
             skip_layers=[])
NETWORK = dict(input_dim=2, output_dim=3, hidden_dim=256, pe_type="encoding", pe_dim=10, mlp_type="origin", mlp_layers=8,
               skip_layers=[4, 7])
GAIN_UV, GAIN_ALPHA = 1.2, 1.8      # default-init networks are nearly constant maps: tracks would barely move
F, LARGER_DIM, KEYFRAME, TIE_DIM = 72, 768, 17, 765
NAMES = [f"p{i}" for i in range(7)]
SOURCE = {f"p{i}": [100 + 90 * i, 150 + 80 * i] for i in range(6)}                      # {name: [y, x]}
TARGET = {f"p{i}": [130 + 78 * i, 125 + 89 * i] for i in range(6) if i not in (2, 4)}
TARGET["q"] = [5, 5]                                                                      # not a source point: ignored
NETWORK_ROWS = 100


def encoded_dim(cfg):
    return 2 * cfg["input_dim"] * cfg["pe_dim"] if cfg["pe_type"] == "encoding" else cfg["input_dim"]


def layer_shapes(cfg):
    """[(out, in)] of hidden.{i}.weight."""
    E, H, L = encoded_dim(cfg), cfg["hidden_dim"], cfg["mlp_layers"]
    return [(cfg["output_dim"] if i == L - 1 else H, E if i == 0 else H + E if i in cfg["skip_layers"] else H)
            for i in range(L)]


def seeded_imlp(cfg, seed, gain=1.0):
    """Shared with the tests: an IMLP_Hash state dict from a CPU generator, weights N(0, gain^2 / fan_in), biases
    N(0, 0.01)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for i, (n, k) in enumerate(layer_shapes(cfg)):
        sd[f"hidden.{i}.weight"] = torch.randn((n, k), generator=g) * (gain / math.sqrt(k))
        sd[f"hidden.{i}.bias"] = torch.randn((n,), generator=g) * 0.1
    return sd


def nets_for(seed):
    """(FG, FG_inverse, F_Alpha) state dicts of a search seed."""
    return (seeded_imlp(FG, 3 * seed, GAIN_UV), seeded_imlp(FG_INV, 3 * seed + 1, GAIN_UV),
            seeded_imlp(ALPHA, 3 * seed + 2, GAIN_ALPHA))


def tie_nets(nets):
    """The inverse network's x and y outputs zeroed (rows 0, 1 of its last layer): every warp is tanh(0) = 0 plus a drag
    through a zero Jacobian, while t, and so alpha, still varies over the frames."""
    inv = dict(nets[1])
    L = FG_INV["mlp_layers"] - 1
    inv[f"hidden.{L}.weight"] = inv[f"hidden.{L}.weight"].clone()
    inv[f"hidden.{L}.bias"] = inv[f"hidden.{L}.bias"].clone()
    inv[f"hidden.{L}.weight"][:2] = 0
    inv[f"hidden.{L}.bias"][:2] = 0
    return nets[0], inv, nets[2]


def threshold_nets(nets):
    """F_Alpha's last layer zeroed: alpha is exactly 0, 0.5 (alpha + 1) exactly the threshold, and no frame is visible."""
    al = dict(nets[2])
    L = ALPHA["mlp_layers"] - 1
    al[f"hidden.{L}.weight"] = torch.zeros_like(al[f"hidden.{L}.weight"])
    al[f"hidden.{L}.bias"] = torch.zeros_like(al[f"hidden.{L}.bias"])
    return nets[0], nets[1], al


def source_tap():
    """Shared with the tests: the TAP dict the propagation edits (tracks of 7 points over F frames)."""
    g = torch.Generator().manual_seed(5)
    return {"pred_tracks": torch.rand((F, len(NAMES), 2), generator=g) * 700,
            "point_name2id": {n: i for i, n in enumerate(NAMES)},
            "point_embedding": torch.zeros((len(NAMES), 8))}


def network_input():
    return torch.rand((NETWORK_ROWS, NETWORK["input_dim"]), generator=torch.Generator().manual_seed(11)) * 2 - 1


# ------------------------------------------------------------------------------------------------------------ reference
def _stub_modules():
    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        return m

    class _OmegaConf:
        @staticmethod
        def load(*a, **k):
            raise NotImplementedError

    return {"tinycudann": mod("tinycudann"), "imageio": mod("imageio"),
            "omegaconf": mod("omegaconf", OmegaConf=_OmegaConf)}


def import_reference():
    if not REFERENCE_ROOT or not os.path.isdir(REFERENCE_ROOT):
        raise SystemExit("set VIDEOSWAP_REFERENCE to a checkout of the reference")
    sys.path.insert(0, REFERENCE_ROOT)
    saved = {k: sys.modules.get(k) for k in _stub_modules()}
    sys.modules.update(_stub_modules())
    try:
        import propagate_point_displacement as ppd
        from videoswap.atlas import implicit_neural_networks as inn
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    ppd.device = "cpu"
    return ppd, inn


class _Recorder:
    def __init__(self, fn, log):
        self.fn, self.log = fn, log

    def __call__(self, *a, **k):
        out = self.fn(*a, **k)
        self.log.append(([x.detach().clone() if torch.is_tensor(x) else x for x in a], out.detach().clone()))
        return out


def run_reference(ppd, inn, nets, larger_dim, tmp):
    """propagate_point_sequence on the CPU with every network call recorded.  Returns (TAP dict, stages)."""
    models = []
    for cfg, sd in zip((FG, FG_INV, ALPHA), nets):
        m = inn.IMLP_Hash(**cfg)
        m.load_state_dict(sd, strict=True)
        models.append(m.eval())
    logs = {k: [] for k in ("fg", "inv", "alpha", "wm", "pp")}
    fg, inv, al = (_Recorder(m, logs[k]) for m, k in zip(models, ("fg", "inv", "alpha")))
    wm0, pp0 = ppd.compute_Wm, ppd.propogate_point
    ppd.compute_Wm, ppd.propogate_point = _Recorder(wm0, logs["wm"]), _Recorder(pp0, logs["pp"])
    src_path = os.path.join(tmp, f"{KEYFRAME:05d}.json")
    tgt_path = os.path.join(tmp, "00017_edit.json")
    tap_path = os.path.join(tmp, "TAP.pth")
    with open(src_path, "w") as f:
        json.dump(SOURCE, f)
    with open(tgt_path, "w") as f:
        json.dump(TARGET, f)
    torch.save(source_tap(), tap_path)
    import numpy as np
    ld = np.maximum(larger_dim, 448)          # np.maximum(res_y, res_x), as process_displacement_propagation
    try:
        with torch.no_grad():
            out = ppd.propagate_point_sequence(
                source_point_path=src_path, source_tap_path=tap_path, target_point_path=tgt_path,
                FG_UV_Mapping=fg, FG_UV_Mapping_Inverse=inv, F_Alpha=al, larger_dim=ld, number_of_frames=F,
                norm_Scoord_func=lambda x: x / (ld / 2) - 1, norm_Tcoord_func=lambda x: x / (F / 2) - 1)
    finally:
        ppd.compute_Wm, ppd.propogate_point = wm0, pp0
    P = len(logs["alpha"])
    fgc = [logs["fg"][5 * p:5 * p + 5] for p in range(P)]       # src, propogate_point's xyt, compute_Wm's 3
    invc = [logs["inv"][4 * p:4 * p + 4] for p in range(P)]     # base rows, compute_Wm's 3
    for p in range(P):
        assert torch.equal(fgc[p][0][1], fgc[p][2][1]) and torch.equal(invc[p][0][1], invc[p][1][1])
    st = {
        "fg_in": torch.cat([torch.cat([fgc[p][2 + s][0][0] for p in range(P)]) for s in range(3)]),
        "fg_out": torch.cat([torch.cat([fgc[p][2 + s][1] for p in range(P)]) for s in range(3)]),
        "J_fg": torch.cat([logs["wm"][2 * p][1] for p in range(P)]),
        "inv_in": torch.cat([torch.cat([invc[p][1 + s][0][0] for p in range(P)]) for s in range(3)]),
        "inv_out": torch.cat([torch.cat([invc[p][1 + s][1] for p in range(P)]) for s in range(3)]),
        "J_inv": torch.cat([logs["wm"][2 * p + 1][1][..., :2] for p in range(P)]),
        "alpha": torch.cat([logs["alpha"][p][1][:, 0] for p in range(P)]),
        "alpha_in": torch.cat([logs["alpha"][p][0][0] for p in range(P)]),
        "dxy": torch.cat([logs["pp"][p][1] for p in range(P)]),
    }
    st["warp"] = torch.cat([invc[p][0][1][:, :2] + logs["pp"][p][1] for p in range(P)])
    return out, st


def margins(st, larger_dim):
    """(least distance of a written coordinate from a half-integer in px, least |0.5 (alpha + 1) - 0.5|)."""
    vis = 0.5 * (st["alpha"] + 1.0) > 0.5
    px = ((st["warp"] + 1) / 2 * larger_dim)[vis].double()
    d = ((px - px.floor()) - 0.5).abs()
    return float(d.min()) if d.numel() else 0.5, float((0.5 * (st["alpha"].double() + 1.0) - 0.5).abs().min())


def acceptable(st, P):
    vis = (0.5 * (st["alpha"] + 1.0) > 0.5).view(P, F)
    frac = vis.float().mean(1)
    motion = (st["warp"].view(P, F, 2).amax(1) - st["warp"].view(P, F, 2).amin(1)).amax(1) * LARGER_DIM / 2
    m_px, m_a = margins(st, LARGER_DIM)
    return bool((frac > 0.1).all() and (frac < 0.9).all() and (motion >= 20).all() and m_px >= 0.01 and m_a >= 1e-4)


def main():
    ppd, inn = import_reference()
    torch.manual_seed(0)
    with tempfile.TemporaryDirectory() as tmp:
        P = sum(1 for k in SOURCE if k in TARGET)
        for seed in range(1000):
            nets = nets_for(seed)
            out, st = run_reference(ppd, inn, nets, LARGER_DIM, tmp)
            if acceptable(st, P):
                break
        else:
            raise SystemExit("no seed below 1000 satisfies the margins")
        print("seed", seed, "margins (px, alpha)", margins(st, LARGER_DIM))
        tie_out, tie_st = run_reference(ppd, inn, tie_nets(nets), TIE_DIM, tmp)
        vis = 0.5 * (tie_st["alpha"] + 1.0) > 0.5
        assert (tie_st["warp"] == 0).all() and vis.any() and (~vis).any()
        thr_out, thr_st = run_reference(ppd, inn, threshold_nets(nets), LARGER_DIM, tmp)
        assert (thr_st["alpha"] == 0).all()
    net = inn.IMLP_Hash(**NETWORK)
    net.load_state_dict(seeded_imlp(NETWORK, 7), strict=True)
    with torch.no_grad():
        net_out = net(network_input())
    gold = {
        "configs": {"FG_UV_Mapping": FG, "FG_UV_Mapping_Inverse": FG_INV, "F_Alpha": ALPHA, "network": NETWORK},
        "seed": seed, "F": F, "larger_dim": LARGER_DIM, "keyframe": KEYFRAME, "source": copy.deepcopy(SOURCE),
        "target": copy.deepcopy(TARGET), "stages": st, "pred_tracks": out["pred_tracks"],
        "tie": {"larger_dim": TIE_DIM, "pred_tracks": tie_out["pred_tracks"], "alpha": tie_st["alpha"]},
        "threshold": {"pred_tracks": thr_out["pred_tracks"]},
        "network": {"seed": 7, "out": net_out},
    }
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, "atlas.pt")
    torch.save(gold, path)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
