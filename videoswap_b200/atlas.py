"""Point-drag propagation on the native path: the reference's propagate_point_displacement.py, which carries the drags
of a few semantic points on one keyframe to every frame through the video's layered neural atlas and returns the edited
TAP dict (the `tap_path` of a shape-changing edit; formats.load_tap reads it).

Only three atlas networks take part: FG_UV_Mapping (x, y, t -> u, v), FG_UV_Mapping_Inverse (u, v, t -> x, y, t) and
F_Alpha (x, y, t -> alpha), all IMLP_Hash MLPs with mlp_type 'origin'.  vs_imlp_forward runs one network in one launch
(fp32 on the CUDA cores) and vs_atlas_propagate runs the whole propagation of all edited points in six launches with no
host sync before the tracks are copied back.  The reference's rules are kept exactly, quirks included:

  * JSON points are {name: [y, x]}.  The keyframe index is int() of the source point file's base name.  Only source
    points that the target file names move; target names that are not source points are ignored; every other track is
    returned unchanged.
  * Coordinates are normalised in Python doubles, x / (larger_dim / 2) - 1, and the drag as the difference of two such
    doubles, each rounded to fp32 once; the keyframe time likewise, t / (F / 2) - 1.  The frame axis is
    torch.arange(F) / (F / 2) - 1 in fp32 (a correctly rounded divide by fp32(F / 2), then the subtract), so the keyframe's
    own t in the forward map can differ from the frame axis at the keyframe in the last bit.
  * compute_Wm's finite differences: steps 0.1 in x (u) and 0.05 in y (v), (f(x + d) - f(x)) / d in fp32.  The drag in uv
    space is dx_dy @ J_fg; per frame the offset is delta_uv @ J_inv with J_inv the x / y columns of the inverse Jacobian.
  * F_Alpha is evaluated at the inverse network's predicted (x, y, t), not at the frame's own t.
  * A frame is visible iff 0.5 (alpha + 1) > 0.5 (strictly).  The edited point's column is cleared to -1 first; visible
    frames get round((w + 1) / 2 larger_dim) with torch.round's half-to-even.
  * The reference evaluates FG(xyt) and the inverse base rows twice with identical inputs; here each is evaluated once.

One deliberate difference: atlas_dims reads only the number of files in frame_path and the configured resolution, where
the reference's load_input_data also reads every frame, mask and flow.  The two numbers propagation takes from it are the
same, and the mask and flow directories need not exist.
"""
from __future__ import annotations

import ctypes as C
import json
import os
from typing import Optional

import torch

from . import _lib
from .formats import _load

_NEEDS_TCNN = "needs tinycudann; point propagation does not use it (only F_Atlas does)"


class IMLP_Hash:
    """implicit_neural_networks.IMLP_Hash with pe_type 'none' / 'encoding' and mlp_type 'origin': fp32 device parameters
    under the reference's keys (hidden.{i}.weight / .bias), a strict load_state_dict and __call__(x [N, in]) -> [N, out]."""

    def __init__(self, input_dim, output_dim, hidden_dim=256, pe_type="none", pe_dim=10, mlp_type="origin",
                 skip_layers=(), mlp_layers=8, use_tanh=True, fp16=False, device="cuda"):
        if pe_type == "hash_encoding":
            raise NotImplementedError(f"pe_type 'hash_encoding' {_NEEDS_TCNN}")
        if mlp_type == "tcnn":
            raise NotImplementedError(f"mlp_type 'tcnn' {_NEEDS_TCNN}")
        if pe_type not in ("none", "encoding") or mlp_type != "origin":
            raise NotImplementedError(f"pe_type {pe_type!r} / mlp_type {mlp_type!r}")
        self.input_dim, self.output_dim, self.hidden_dim = int(input_dim), int(output_dim), int(hidden_dim)
        self.pe_type, self.pe_dim, self.mlp_layers = pe_type, int(pe_dim), int(mlp_layers)
        self.skip_layers, self.use_tanh = [int(i) for i in skip_layers], bool(use_tanh)
        if self.mlp_layers < 1 or any(not 1 <= i < self.mlp_layers for i in self.skip_layers):
            raise ValueError(f"mlp_layers {mlp_layers} / skip_layers {list(skip_layers)}: every skip layer must be in "
                             f"[1, mlp_layers)")
        self.device = torch.device(device)
        E = 2 * self.input_dim * self.pe_dim if pe_type == "encoding" else self.input_dim
        L, H = self.mlp_layers, self.hidden_dim
        self.shapes = {}
        for i in range(L):
            k = E if i == 0 else H + E if i in self.skip_layers else H
            n = self.output_dim if i == L - 1 else H
            self.shapes[f"hidden.{i}.weight"], self.shapes[f"hidden.{i}.bias"] = (n, k), (n,)
        self.params = {k: torch.zeros(s, dtype=torch.float32, device=self.device) for k, s in self.shapes.items()}
        self._pack()

    def state_dict(self):
        return dict(self.params)

    def load_state_dict(self, sd, strict=True):
        """Strict: the keys and shapes must be exactly the reference's."""
        missing, extra = sorted(set(self.shapes) - set(sd)), sorted(set(sd) - set(self.shapes))
        if missing or extra:
            raise KeyError(f"IMLP_Hash state dict: missing {missing}, unexpected {extra}")
        for k, s in self.shapes.items():
            if tuple(sd[k].shape) != s:
                raise ValueError(f"IMLP_Hash state dict: {k} has shape {tuple(sd[k].shape)}, expected {s}")
        self.params = {k: torch.as_tensor(sd[k]).detach().to(self.device, torch.float32).contiguous() for k in self.shapes}
        self._pack()

    def _pack(self):
        parts = []
        for i in range(self.mlp_layers):
            parts += [self.params[f"hidden.{i}.weight"].t().reshape(-1), self.params[f"hidden.{i}.bias"]]
        self.packed = torch.cat(parts).contiguous()

    def desc(self) -> _lib.ImlpDescStruct:
        mask = 0
        for i in self.skip_layers:
            mask |= 1 << i
        return _lib.ImlpDescStruct(C.c_void_p(self.packed.data_ptr()), self.input_dim, self.output_dim, self.hidden_dim,
                                   self.mlp_layers, self.pe_dim if self.pe_type == "encoding" else 0, mask,
                                   int(self.use_tanh))

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        if self.device.type != "cuda":
            raise RuntimeError("IMLP_Hash runs on a CUDA device only (there is no CPU path)")
        x = x.to(self.device, torch.float32).contiguous()
        if x.dim() != 2 or x.shape[1] != self.input_dim:
            raise ValueError(f"expected [N, {self.input_dim}] inputs, got {tuple(x.shape)}")
        out = torch.empty((x.shape[0], self.output_dim), dtype=torch.float32, device=self.device)
        if x.shape[0]:
            d = self.desc()
            _lib.call("vs_imlp_forward", torch.cuda.current_stream(self.device).cuda_stream, C.byref(d),
                      C.c_void_p(x.data_ptr()), int(x.shape[0]), C.c_void_p(out.data_ptr()))
        return out

    forward = __call__


def init_atlas_model(atlas_config: dict, atlas_model, device="cuda"):
    """(FG_UV_Mapping, FG_UV_Mapping_Inverse, F_Alpha) from a checkpoint {'FG_UV_Mapping': sd, ...} (a path or a loaded
    dict) as train_atlas.py writes it, built from atlas_config['models']."""
    ckpt = _load(atlas_model)
    nets = []
    for name in ("FG_UV_Mapping", "FG_UV_Mapping_Inverse", "F_Alpha"):
        net = IMLP_Hash(**atlas_config["models"][name], device=device)
        net.load_state_dict(ckpt[name])
        nets.append(net)
    return tuple(nets)


def atlas_dims(datasets_opt: dict):
    """(number_of_frames, larger_dim) as load_input_data gives them: min(max_frames, number of files in frame_path) and
    max(res_x, res_y).  Reads no image and needs no mask or flow directory (the reference reads them all; the two
    numbers are the same)."""
    n = len(os.listdir(datasets_opt["frame_path"]))
    return int(min(int(datasets_opt["max_frames"]), n)), int(max(int(datasets_opt["res_x"]), int(datasets_opt["res_y"])))


def _points(obj):
    if isinstance(obj, (str, os.PathLike)):
        with open(obj) as f:
            return json.load(f)
    return obj


def propagate_point_sequence(source_point, source_tap, target_point, FG_UV_Mapping, FG_UV_Mapping_Inverse, F_Alpha,
                             larger_dim: int, number_of_frames: int, keyframe: Optional[int] = None) -> dict:
    """The edited TAP dict: source_point / target_point JSON files {name: [y, x]} (or dicts), source_tap a TAP file (or
    dict).  The keyframe is int() of the source file's base name unless given.  Returns a new dict whose pred_tracks
    (on the CPU, in the input's dtype) has the moved points' columns replaced; the input is not modified."""
    if keyframe is None:
        if not isinstance(source_point, (str, os.PathLike)):
            raise ValueError("keyframe must be given when source_point is not a file named after its frame")
        keyframe = int(os.path.splitext(os.path.basename(os.fspath(source_point)))[0])
    src, tgt = _points(source_point), _points(target_point)
    tap = _load(source_tap)
    tracks = torch.as_tensor(tap["pred_tracks"]).detach().cpu().clone()
    name2id = tap["point_name2id"]
    F, ld = int(number_of_frames), int(larger_dim)
    moved = [(name2id[k], v, tgt[k]) for k, v in src.items() if k in tgt]
    if tracks.dim() != 3 or tracks.shape[0] != F or tracks.shape[2] != 2:
        raise ValueError(f"pred_tracks must be [{F}, P, 2] for number_of_frames = {F}, got {tuple(tracks.shape)}")
    if moved:
        s = ld / 2
        pts = torch.tensor([[sx / s - 1, sy / s - 1, (tx / s - 1) - (sx / s - 1), (ty / s - 1) - (sy / s - 1)]
                            for _, (sy, sx), (ty, tx) in moved], dtype=torch.float64).float()
        t_key = float(torch.tensor(keyframe / (F / 2) - 1, dtype=torch.float64).float())
        res, _ = propagate_points((FG_UV_Mapping, FG_UV_Mapping_Inverse, F_Alpha), pts, t_key, F, ld)
        res = res.cpu()
        for p, (col, _, _) in enumerate(moved):
            tracks[:, col] = res[:, p].to(tracks.dtype)
    out = dict(tap)
    out["pred_tracks"] = tracks
    return out


def propagate_points(nets, pts: torch.Tensor, t_key: float, F: int, larger_dim: int):
    """vs_atlas_propagate: nets (FG_UV_Mapping, FG_UV_Mapping_Inverse, F_Alpha), pts fp32 [P, 4] = normalised (x, y, dx,
    dy), t_key the normalised keyframe time -> (tracks fp32 [F, P, 2] on the device, -1 where occluded, and the
    workspace with the stages; see `stages`).  Asynchronous on the current stream."""
    dev = nets[0].device
    if dev.type != "cuda" or any(n.device != dev for n in nets):
        raise RuntimeError("the three networks must be on one CUDA device")
    P = int(pts.shape[0])
    d_pts = pts.to(dev, torch.float32).contiguous()
    ws = torch.empty((21 * P + 25 * P * F,), dtype=torch.float32, device=dev)
    res = torch.empty((F, P, 2), dtype=torch.float32, device=dev)
    descs = [n.desc() for n in nets]
    _lib.call("vs_atlas_propagate", torch.cuda.current_stream(dev).cuda_stream, *[C.byref(d) for d in descs],
              C.c_void_p(d_pts.data_ptr()), float(t_key), P, int(F), int(larger_dim), C.c_void_p(ws.data_ptr()),
              C.c_void_p(res.data_ptr()))
    return res, ws


def stages(ws: torch.Tensor, P: int, F: int) -> dict:
    """Views of vs_atlas_propagate's workspace (the header's layout)."""
    names = [("fg_in", (3 * P, 3)), ("fg_out", (3 * P, 2)), ("J_fg", (P, 2, 2)), ("delta_uv", (P, 2)),
             ("inv_in", (3 * P * F, 3)), ("inv_out", (3 * P * F, 3)), ("alpha", (P * F,)), ("J_inv", (P * F, 2, 2)),
             ("warp", (P * F, 2))]
    out, o = {}, 0
    for k, s in names:
        n = 1
        for d in s:
            n *= d
        out[k] = ws[o:o + n].view(s)
        o += n
    return out


def process_displacement_propagation(atlas_config, atlas_model, source_tap, source_point, target_point, device="cuda"):
    """The reference's entry point: atlas_config a dict or a YAML file, atlas_model a checkpoint path or dict."""
    if isinstance(atlas_config, (str, os.PathLike)):
        import yaml
        with open(atlas_config) as f:
            atlas_config = yaml.safe_load(f)
    nets = init_atlas_model(atlas_config, atlas_model, device=device)
    F, ld = atlas_dims(atlas_config["datasets"])
    return propagate_point_sequence(source_point, source_tap, target_point, *nets, larger_dim=ld, number_of_frames=F)
