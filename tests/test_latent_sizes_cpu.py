"""CPU tests for latents whose height or width is not a multiple of 8: the oracle restatement must reproduce the fixtures
that oracle/make_golden_sizes.py generated with the REFERENCE's own model files (its forward_upsample_size path)."""
import os

import pytest
import torch

from oracle import unet3d_oracle as O
from oracle import sized as S
from oracle.make_golden import CASES as SQUARE_CASES
from oracle.make_golden import make_inputs as square_inputs
from oracle.make_golden_sizes import CASES, make_inputs
from oracle.sized import level_sizes
from videoswap_b200.spec import UNetConfig, unet_param_shapes
from videoswap_b200.weights import seeded_state_dict

GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.mark.parametrize("name", ["tiny_odd", "full_arch_odd"])
def test_unet_oracle_matches_reference_golden_odd_sizes(name):
    g = torch.load(os.path.join(GOLD, f"unet_{name}.pt"))
    case = g["case"]
    assert case == CASES[name]
    cfg = UNetConfig(block_out_channels=case["boc"], cross_attention_dim=case["ctx"], norm_num_groups=case["groups"])
    sd = seeded_state_dict(unet_param_shapes(cfg), seed=0)
    wsum = float(sum(v.double().sum() for k, v in sd.items() if not k.endswith(".pe")))
    assert abs(wsum - g["weights_checksum"]) < 1e-6 * abs(wsum), "seeded weights differ from the golden run"
    x, ehs, res = make_inputs(case)
    assert tuple(x.shape[-2:]) == (case["h"], case["w"])
    assert [tuple(r.shape[-2:]) for r in res] == level_sizes(case["h"], case["w"])
    ocfg = O.OracleConfig(block_out_channels=case["boc"], cross_attention_dim=case["ctx"], norm_groups=case["groups"])
    with torch.no_grad():
        out = S.unet_forward(sd, ocfg, x, case["t"], ehs, res)
    assert out.shape == g["out"].shape
    err = (out - g["out"]).abs().max().item()
    assert err < 2e-4, err


def test_sized_oracle_is_the_oracle_at_multiples_of_8():
    """At multiples of 8 every up-sampler targets exactly 2x: the sized oracle computes bit for bit what the oracle does."""
    case = SQUARE_CASES["tiny_edlora_res"]
    cfg = UNetConfig(block_out_channels=case["boc"], cross_attention_dim=case["ctx"], norm_num_groups=case["groups"])
    sd = seeded_state_dict(unet_param_shapes(cfg), seed=0)
    ocfg = O.OracleConfig(block_out_channels=case["boc"], cross_attention_dim=case["ctx"], norm_groups=case["groups"])
    x, ehs, res = square_inputs(case)
    with torch.no_grad():
        a = O.unet_forward(sd, ocfg, x, case["t"], ehs, res)
        b = S.unet_forward(sd, ocfg, x, case["t"], ehs, res)
    assert torch.equal(a, b)
    assert O.unet_forward.__name__ == "unet_forward" and O._conv_per_frame.__name__ == "_conv_per_frame"   # restored


def test_level_sizes_follow_the_stride2_conv():
    """The ceil chain is what a 3x3, stride-2, pad-1 conv produces; at multiples of 8 it is the halving chain."""
    for h, w in [(45, 60), (90, 160), (9, 13), (3, 5), (1, 1), (56, 96)]:
        x = torch.zeros(1, 1, h, w)
        sizes = [(h, w)]
        for _ in range(3):
            x = torch.nn.functional.conv2d(x, torch.zeros(1, 1, 3, 3), stride=2, padding=1)
            sizes.append(tuple(x.shape[-2:]))
        assert level_sizes(h, w) == sizes
    assert level_sizes(64, 64) == [(64 >> l, 64 >> l) for l in range(4)]


def test_nearest_to_odd_size_drops_the_last_row():
    """torch's nearest to 2n - 1 is 2x nearest without the last row / column (what the sub-pixel conv relies on)."""
    for n in (1, 2, 3, 7, 12, 23):
        x = torch.randn(1, 2, n, n + 1)
        up = torch.nn.functional.interpolate(x, size=(2 * n - 1, 2 * n + 1), mode="nearest")
        up2 = torch.nn.functional.interpolate(x, scale_factor=2.0, mode="nearest")
        assert torch.equal(up, up2[:, :, :2 * n - 1, :2 * n + 1])
