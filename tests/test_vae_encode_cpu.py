"""CPU tests of the VAE encoder's host side and of the stride-2 down-sampler's addressing: the encode-side state_dict
surface against the oracle's restatement of diffusers 0.19.3, old attention names, decoder-only and partial-encoder dicts,
shape errors; the oracle's right / bottom padding; and a torch emulation of the kernel's parity-view reads that passes the
GPU test's per-element comparator while each planted addressing bug fails it."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import videoswap_b200 as V
from tests import downsample_checks as D
from tests import vae_encoder_oracle as EO
from videoswap_b200 import vae as VAE


def _full(seed=7):
    cfg = V.VAEConfig()
    return V.seeded_state_dict({**V.vae_param_shapes(cfg), **V.vae_encoder_param_shapes(cfg)}, seed=seed)


# ---------------------------------------------------------------------------------------------------- keys
def test_encoder_keys_and_shapes_match_the_oracle():
    shapes = V.vae_encoder_param_shapes(V.VAEConfig())
    assert dict(shapes) == dict(EO.param_shapes())
    assert sum(int(np.prod(s)) for s in shapes.values()) == 34_163_664     # + 49_490_199 (decoder) = 83_653_863
    assert sum(1 for k in shapes if k.endswith("conv_shortcut.weight")) == 2           # down blocks 1 and 2, first resnet
    assert sum(1 for k in shapes if ".downsamplers.0.conv.weight" in k) == 3
    assert not set(shapes) & set(V.vae_param_shapes(V.VAEConfig()))                     # the decoder list stays decoder-only


def test_old_encoder_attention_names_give_the_same_weights():
    cfg = V.VAEConfig()
    new = _full()
    a = "encoder.mid_block.attentions.0"
    old = {}
    for k, v in new.items():
        for o, n in VAE._OLD_ATTN.items():
            if k.startswith(f"{a}.{n}."):
                leaf = k.rsplit(".", 1)[1]
                k = f"{a}.{o}.{leaf}"
                if leaf == "weight":
                    v = v[..., None, None]
                break
        old[k] = v
    assert f"{a}.query.weight" in old and old[f"{a}.proj_attn.weight"].shape == (512, 512, 1, 1)
    e_new, e_old = VAE.convert_encoder_state_dict(new, cfg), VAE.convert_encoder_state_dict(old, cfg)
    assert e_new.keys() == e_old.keys() == set(V.vae_encoder_param_shapes(cfg))
    assert all(torch.equal(e_new[k], e_old[k]) for k in e_new)
    d_new, d_old = VAE.convert_state_dict(new, cfg), VAE.convert_state_dict(old, cfg)    # decoder unaffected
    assert all(torch.equal(d_new[k], d_old[k]) for k in d_new)
    with pytest.raises(KeyError, match="twice"):
        VAE.convert_encoder_state_dict({**new, f"{a}.key.bias": torch.zeros(512)}, cfg)


def test_decoder_only_and_partial_encoder_dicts():
    cfg = V.VAEConfig()
    dec = V.seeded_state_dict(V.vae_param_shapes(cfg), seed=7)
    out, missing = VAE._convert_half(dec, V.vae_encoder_param_shapes(cfg), VAE._ENCODER_ATTN)
    assert out == {} and missing == list(V.vae_encoder_param_shapes(cfg))
    with pytest.raises(KeyError, match="missing encoder keys"):
        VAE.convert_encoder_state_dict(dec, cfg)
    partial = {**dec, "encoder.conv_in.weight": torch.zeros(128, 3, 3, 3), "quant_conv.weight": torch.zeros(8, 8, 1, 1)}
    out, missing = VAE._convert_half(partial, V.vae_encoder_param_shapes(cfg), VAE._ENCODER_ATTN)
    assert set(out) == {"encoder.conv_in.weight", "quant_conv.weight"} and "encoder.conv_in.bias" in missing
    with pytest.raises(KeyError, match="encoder.conv_in.bias"):
        VAE.convert_encoder_state_dict(partial, cfg)
    assert VAE.convert_state_dict(partial, cfg).keys() == VAE.convert_state_dict(dec, cfg).keys()


def test_encoder_shape_and_unknown_key_errors():
    cfg = V.VAEConfig()
    sd = _full()
    with pytest.raises(ValueError, match="shape"):
        VAE.convert_encoder_state_dict({**sd, "encoder.conv_in.weight": torch.zeros(128, 4, 3, 3)}, cfg)
    with pytest.raises(ValueError, match="shape"):
        VAE.convert_encoder_state_dict({**sd, "quant_conv.weight": torch.zeros(4, 4, 1, 1)}, cfg)
    with pytest.raises(KeyError, match="unexpected"):
        VAE.convert_encoder_state_dict({**sd, "encoder.down_blocks.3.downsamplers.0.conv.weight": torch.zeros(512, 512, 3, 3)}, cfg)


# ---------------------------------------------------------------------------------------------------- down-sampler
def test_oracle_downsample_pads_right_and_bottom_only():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 5, 6, 10, generator=g)
    sd = {"d.conv.weight": torch.randn(7, 5, 3, 3, generator=g), "d.conv.bias": torch.randn(7, generator=g)}
    out = EO.downsample(x, sd, "d")
    assert tuple(out.shape) == (2, 7, 3, 5)
    ref = F.conv2d(F.pad(x, (0, 1, 0, 1)), sd["d.conv.weight"], sd["d.conv.bias"], stride=2)
    assert torch.equal(out, ref)
    # the same sum written out tap by tap: out[y, x] = b + sum_{dy, dx} w[:, :, dy, dx] x[2y + dy, 2x + dx] (0 past the end)
    xp = torch.zeros(2, 5, 7, 11)
    xp[:, :, :6, :10] = x
    taps = sum(torch.einsum("nchw,oc->nohw", xp[:, :, dy:dy + 6:2, dx:dx + 10:2], sd["d.conv.weight"][:, :, dy, dx])
               for dy in range(3) for dx in range(3))
    assert torch.allclose(out, taps + sd["d.conv.bias"][:, None, None], atol=1e-5)
    sym = F.conv2d(x, sd["d.conv.weight"], sd["d.conv.bias"], stride=2, padding=1)      # the UNet's geometry differs
    assert sym.shape == out.shape and not torch.allclose(sym, out, atol=1e-2)


CASES = [(2, 8, 8, 64, 32), (3, 6, 10, 64, 64), (1, 16, 12, 128, 32)]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "x".join(map(str, c)))
def test_parity_view_emulation_passes_and_planted_bugs_fail(case):
    n, H, W, C, co = case
    w, b = D.weights(co, C, seed=H * W)
    wp = D.pack(w)
    for kind, x in (("impulse", D.probe_input(n, H, W, C, seed=1)),
                    ("random", torch.randn(n, H, W, C, generator=torch.Generator().manual_seed(2)).half())):
        err, _ = D.compare(D.emulate(x, wp, b), x, w, b)
        print(f"\n{case} {kind}: emulation worst err / bound {err:.3g}")
        assert err <= 1.0, (kind, err)
        im = D.im2col(x).float() @ wp.float().t() + b.float()
        assert torch.equal(im.half().reshape(n, H // 2, W // 2, co), D.emulate(x, wp, b))   # same K order as the im2col GEMM
        for bug in D.PLANTED:
            err, where = D.compare(D.emulate(x, wp, b, bug=bug), x, w, b)
            print(f"  planted {bug}: worst err / bound {err:.3g}")
            assert err > 1.0, f"{kind}: planted bug {bug} passes the comparator"
