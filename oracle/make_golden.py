"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/*.pt by running the REFERENCE's own model files
(a checkout of the reference, through oracle/diffusers_stub) on seeded inputs and seeded weights
(videoswap_b200.weights.seeded_state_dict).  Run where the reference tree is checked out:  python -m oracle.make_golden
The fixtures pin oracle/unet3d_oracle.py (tests/test_oracle_golden.py) wherever the reference is absent."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.ref_loader import build_reference_unet, load_reference  # noqa: E402
from videoswap_b200.spec import UNetConfig, adapter_param_shapes, unet_param_shapes  # noqa: E402
from videoswap_b200.weights import seeded_state_dict  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def randn(shape, seed):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed))


def make_inputs(case):
    """Shared by the golden maker and the tests: everything is derived from seeds."""
    b, f, hw = case["batch"], case["frames"], case["hw"]
    x = randn((b, 4, f, hw, hw), 2)
    if case["edlora"]:
        ehs = randn((b, 16, 77, case["ctx"]), 3)
    else:
        ehs = randn((b, 77, case["ctx"]), 3)
    res = None
    if case["residuals"]:
        boc = case["boc"]
        res = [0.5 * randn((b * f, c, max(hw >> l, 1), max(hw >> l, 1)), 10 + l) for l, c in enumerate(boc)]
    return x, ehs, res


CASES = {
    "tiny_edlora_res": dict(boc=(32, 64, 128, 128), ctx=64, groups=8, batch=2, frames=3, hw=8, edlora=True,
                            residuals=True, t=981, pe=24),
    "tiny_plain": dict(boc=(32, 64, 128, 128), ctx=64, groups=8, batch=1, frames=2, hw=16, edlora=False,
                       residuals=False, t=501, pe=24),
    "full_arch_small": dict(boc=(320, 640, 1280, 1280), ctx=768, groups=32, batch=1, frames=2, hw=8, edlora=True,
                            residuals=False, t=981, pe=24),
    # BASELINE configs[0] ("single DDIM step, 1-frame 64x64 latent") at its real size, with ED-LoRA embeddings and adapter
    # residuals: N = 4096 attention, 64x64 convs, GroupNorm groups of 40 960 elements
    "full_arch_c1": dict(boc=(320, 640, 1280, 1280), ctx=768, groups=32, batch=1, frames=1, hw=64, edlora=True,
                         residuals=True, t=981, pe=24),
}


def run_case(name, case):
    cfg = UNetConfig(block_out_channels=case["boc"], cross_attention_dim=case["ctx"], norm_num_groups=case["groups"],
                     temporal_position_encoding_max_len=case["pe"])
    sd = seeded_state_dict(unet_param_shapes(cfg), seed=0)
    model = build_reference_unet(case["boc"], case["ctx"], pe_max_len=case["pe"], norm_num_groups=case["groups"])
    missing, unexpected = model.load_state_dict(sd, strict=True)
    x, ehs, res = make_inputs(case)
    with torch.no_grad():
        out = model(x, case["t"], ehs, down_block_additional_residuals=[r.clone() for r in res] if res else None,
                    return_dict=False)[0]
    wsum = float(sum(v.double().sum() for k, v in sd.items() if not k.endswith(".pe")))
    torch.save({"case": case, "out": out.contiguous(), "weights_checksum": wsum}, os.path.join(OUT, f"unet_{name}.pt"))
    print(name, tuple(out.shape), float(out.std()), wsum)


def run_adapter():
    ns = load_reference()
    shapes = adapter_param_shapes()
    sd = seeded_state_dict(shapes, seed=5)
    ad = ns.SparsePointAdapter().eval()
    ad.load_state_dict(sd)
    g = torch.Generator().manual_seed(4)
    tracks = torch.rand((4, 6, 2), generator=g) * 130 - 1.0       # some < 0 (invisible), some at the far edge
    tracks[0, 0] = torch.tensor([127.9, 127.9])
    tracks[1, 1] = torch.tensor([0.0, 64.5])
    emb = randn((6, 1280), 6)
    with torch.no_grad():
        maps = ad(tracks[None], (128, 128), emb[None], index_list=None)
    torch.save({"tracks": tracks, "emb": emb, "size": (128, 128), "maps_sparse": sparsify(maps)}, os.path.join(OUT, "adapter.pt"))
    print("adapter", [tuple(m.shape) for m in maps], [float(m.abs().sum()) for m in maps])


def adapter_fp16_inputs():
    """Shared with the tests: tracks on a 768x448 frame (the reference's usual size), several beyond 512 px where fp16
    coordinates quantise to 0.5 px, invisible points, exact cell centres and the far edges."""
    g = torch.Generator().manual_seed(14)
    tracks = torch.rand((5, 8, 2), generator=g) * torch.tensor([768.0, 448.0])
    tracks[0, 0] = torch.tensor([767.9, 447.9])
    tracks[1, 1] = torch.tensor([-1.0, 100.0])
    tracks[2, 2] = torch.tensor([600.3, -1.0])
    tracks[3, 3] = torch.tensor([512.0, 256.0])
    tracks[4, 4] = torch.tensor([700.77, 13.31])
    emb = randn((8, 1280), 16)
    return tracks, emb, (768, 448), [0, 1, 2, 3, 4, 6, 7]


def sparsify(maps):
    """The maps are zero except around the points: (frame, y, x) of the non-zero cells and their channel vectors."""
    sparse = []
    for m in maps:
        idx = (m != 0).any(dim=1).nonzero()
        sparse.append({"shape": tuple(m.shape), "idx": idx.to(torch.int32), "val": m[idx[:, 0], :, idx[:, 1], idx[:, 2]].contiguous()})
    return sparse


def densify(sparse):
    out = []
    for s in sparse:
        m = torch.zeros(s["shape"], dtype=s["val"].dtype)
        idx = s["idx"].long()
        m[idx[:, 0], :, idx[:, 1], idx[:, 2]] = s["val"]
        out.append(m)
    return out


def run_adapter_fp16():
    """The reference's inference arithmetic: adapter weights, tracks and embedding all cast to fp16
    (test.py:75-78 `.to(torch.float16)`, pipeline_videoswap.py:528-533), maps accumulated in fp16."""
    ns = load_reference()
    sd = seeded_state_dict(adapter_param_shapes(), seed=5)
    ad = ns.SparsePointAdapter().eval()
    ad.load_state_dict(sd)
    ad = ad.half()
    tracks, emb, size, index_list = adapter_fp16_inputs()
    with torch.no_grad():
        maps = ad(tracks[None].half(), size, emb[None].half(), index_list=index_list)
    assert all(m.dtype == torch.float16 for m in maps)
    torch.save({"maps_sparse": sparsify(maps)}, os.path.join(OUT, "adapter_fp16.pt"))
    print("adapter_fp16", [tuple(m.shape) for m in maps], [float(m.float().abs().sum()) for m in maps])


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    which = sys.argv[1:] or list(CASES) + ["adapter", "adapter_fp16"]
    for n in which:
        if n == "adapter":
            run_adapter()
        elif n == "adapter_fp16":
            run_adapter_fp16()
        else:
            run_case(n, CASES[n])
