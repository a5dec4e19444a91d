"""A torch restatement of the layered-atlas point propagation (the reference's propagate_point_displacement.py with the
IMLP_Hash "origin" MLP), runnable on the CPU or a GPU, for the fixture tests and tools/gpu_atlas_propagate.py.

It batches what the reference computes point by point: FG_UV_Mapping on 3 rows per point, FG_UV_Mapping_Inverse on 3 F
rows per point and F_Alpha on F rows per point.  Each rule the propagation depends on is one small function here, so the
CPU tests can plant a bug in exactly one of them."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as Fn

DX, DY = 0.1, 0.05           # compute_Wm's deltax, deltay


# ---------------------------------------------------------------------------------------------------------------- MLP
def encode(x: torch.Tensor, pe_dim: int) -> torch.Tensor:
    """positionalEncoding_vec: [N, d] -> [N, 2 d pe_dim], frequency-major, sines then cosines of the d inputs."""
    b = torch.tensor([(2 ** j) * math.pi for j in range(pe_dim)], dtype=x.dtype, device=x.device)
    proj = x[:, :, None] * b
    mapped = torch.cat((torch.sin(proj), torch.cos(proj)), 1)
    return mapped.transpose(2, 1).reshape(x.shape[0], -1)


def imlp(sd: dict, cfg: dict, x: torch.Tensor) -> torch.Tensor:
    """IMLP_Hash.forward with pe_type 'none' / 'encoding' and mlp_type 'origin'; sd has the reference's keys."""
    if cfg.get("pe_type", "none") == "encoding":
        x = encode(x, cfg.get("pe_dim", 10))
    inp = x
    skip = cfg.get("skip_layers", [])
    for i in range(cfg.get("mlp_layers", 8)):
        if i > 0:
            x = Fn.relu(x)
        if i in skip:
            x = torch.cat((x, inp), 1)
        x = Fn.linear(x, sd[f"hidden.{i}.weight"], sd[f"hidden.{i}.bias"])
    return torch.tanh(x) if cfg.get("use_tanh", True) else x


# ---------------------------------------------------------------------------------------------------------- propagation
def point_xy(v):
    """A JSON point is [y, x]."""
    y, x = v
    return x, y


def norm_s(v, larger_dim):
    """norm_Scoord_func in Python doubles."""
    return v / (larger_dim / 2) - 1


def frame_axis(F: int, device) -> torch.Tensor:
    """norm_Tcoord_func(torch.arange(F)): fp32."""
    return torch.arange(F, device=device) / (F / 2) - 1


def alpha_input(xyt_pred: torch.Tensor, t_frames: torch.Tensor) -> torch.Tensor:
    """F_Alpha reads the inverse network's predicted (x, y, t), not the frame's own t."""
    return xyt_pred


def visible(alpha: torch.Tensor) -> torch.Tensor:
    return 0.5 * (alpha + 1.0) > 0.5


def to_pixel(w: torch.Tensor, larger_dim) -> torch.Tensor:
    """torch.round (half to even) of (w + 1) / 2 larger_dim."""
    return torch.round((w + 1) / 2 * larger_dim)


def clear_column(tracks: torch.Tensor, col: int):
    tracks[:, col, :] = torch.tensor([-1, -1])


def normalised_points(source_point: dict, target_point: dict, name2id: dict, keyframe: int, larger_dim, F: int):
    """(columns, fp32 [P, 4] = (x, y, dx, dy), fp32 t_key) of the source points that the target file moves, in the source
    file's order: every value a Python double rounded to fp32 once."""
    cols, rows = [], []
    for k, v in source_point.items():
        if k not in target_point:
            continue
        sx, sy = point_xy(v)
        tx, ty = point_xy(target_point[k])
        cols.append(name2id[k])
        rows.append([norm_s(sx, larger_dim), norm_s(sy, larger_dim), norm_s(tx, larger_dim) - norm_s(sx, larger_dim),
                     norm_s(ty, larger_dim) - norm_s(sy, larger_dim)])
    pts = torch.tensor(rows, dtype=torch.float64).float().reshape(-1, 4)
    t_key = torch.tensor(keyframe / (F / 2) - 1, dtype=torch.float64).float()
    return cols, pts, t_key


def propagate(nets, cfgs, pts: torch.Tensor, t_key: torch.Tensor, F: int, larger_dim) -> dict:
    """The stages of propagate_point_sequence for P points at once.  nets / cfgs: (FG, FG_inverse, alpha) state dicts and
    configs on pts' device.  Returns fg_in [3P, 3], fg_out [3P, 2], J_fg [P, 2, 2], delta_uv [P, 2], inv_in [3PF, 3],
    inv_out [3PF, 3], alpha [PF], J_inv [PF, 2, 2], warp [PF, 2], tracks [F, P, 2] (rows p F + f as in the kernels)."""
    fg, inv, al = nets
    cf, ci, ca = cfgs
    dev = pts.device
    P = pts.shape[0]
    xyt = torch.cat([pts[:, :2], t_key.to(dev).expand(P, 1)], 1)
    xp, yp = xyt.clone(), xyt.clone()
    xp[:, 0] = xyt[:, 0] + DX
    yp[:, 1] = xyt[:, 1] + DY
    fg_in = torch.cat([xyt, xp, yp])
    fg_out = imlp(fg, cf, fg_in)
    uv, uvx, uvy = fg_out.view(3, P, 2)
    J_fg = torch.stack([(uvx - uv) / DX, (uvy - uv) / DY], 1)
    delta_uv = pts[:, None, 2:4].bmm(J_fg)[:, 0]
    t = frame_axis(F, dev)
    base = torch.cat([uv[:, None].expand(P, F, 2), t[None, :, None].expand(P, F, 1)], -1).reshape(P * F, 3)
    up, vp = base.clone(), base.clone()
    up[:, 0] = base[:, 0] + DX
    vp[:, 1] = base[:, 1] + DY
    inv_in = torch.cat([base, up, vp])
    inv_out = imlp(inv, ci, inv_in)
    xyt_pred, xu, xv = inv_out.view(3, P * F, 3)
    J_inv = torch.stack([(xu - xyt_pred) / DX, (xv - xyt_pred) / DY], 1)[..., :2]
    warp = xyt_pred[:, :2] + delta_uv.repeat_interleave(F, 0)[:, None].bmm(J_inv)[:, 0]
    alpha = imlp(al, ca, alpha_input(xyt_pred, t.repeat(P)[:, None]))[:, 0]
    px = to_pixel(warp, larger_dim)
    vis = visible(alpha)
    tracks = torch.where(vis[:, None], px, torch.full_like(px, -1.0))
    return dict(fg_in=fg_in, fg_out=fg_out, J_fg=J_fg, delta_uv=delta_uv, inv_in=inv_in, inv_out=inv_out, alpha=alpha,
                J_inv=J_inv, warp=warp, visible=vis.view(P, F).t(), tracks=tracks.view(P, F, 2).transpose(0, 1))


def propagate_tap(nets, cfgs, source_point: dict, source_tap: dict, target_point: dict, keyframe: int, larger_dim,
                  F: int, device="cpu"):
    """(new TAP dict, stages) of propagate_point_sequence on already-loaded inputs."""
    cols, pts, t_key = normalised_points(source_point, target_point, source_tap["point_name2id"], keyframe, larger_dim, F)
    tracks = source_tap["pred_tracks"].clone()
    st = None
    if cols:
        st = propagate(nets, cfgs, pts.to(device), t_key, F, larger_dim)
        res, vis = st["tracks"].cpu(), st["visible"].cpu()
        for p, col in enumerate(cols):
            clear_column(tracks, col)
            tracks[vis[:, p], col] = res[vis[:, p], p].to(tracks.dtype)
    out = dict(source_tap)
    out["pred_tracks"] = tracks
    return out, st
