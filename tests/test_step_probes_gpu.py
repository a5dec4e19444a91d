"""Per-element tests of the denoising step's small kernels (pytest -m gpu), with the probes and bounds of
tests/step_probes.py: the point adapter through `vs_adapter_level` at all four levels (integer-exact MLP, every input
column of both layers, every point row block, the splat at every border, mask, frame and scale, fp16 coordinate
quantisation) and the time embedding through `vs_unet_time_embedding` with distinct timesteps per row; then the whole
UNet with a [B] timestep, per batch element and frame against the oracle."""
import pytest
import torch

from oracle import unet3d_oracle as O
from tests import step_probes as S
from tests import unet_checks as UC
from videoswap_b200 import ops

pytestmark = pytest.mark.gpu


def _adapter(w0, b0, w1, b1, pe, tracks, h, w, rate, mask, coord_fp16, scale):
    return ops.adapter_level(w0, b0, w1, b1, pe, tracks, h, w, rate, mask, coord_fp16, scale)


def _report(name, r):
    print(f"\n{name}: {r['what']} (err {r['err']:.4g})")
    assert r["ok"], f"{name}: {r['what']}"


@pytest.mark.parametrize("level", range(4))
@pytest.mark.parametrize("kind", ["regimes", "dense"])
def test_adapter_mlp_exact_at_cells(level, kind):
    for coord_fp16 in (True, False):
        _report(f"cells L{level} {kind}", S.check_adapter_cells(_adapter, level, 9, kind, coord_fp16=coord_fp16, seed=level))


@pytest.mark.parametrize("P", [1, 7, 8, 9, 33, 200])
def test_adapter_every_k_and_row_block(P):
    """+-1 embeddings over every input column, one-hot second layer; P covers the row loop's first block, its boundary
    and later blocks; the 1278 / 98 widths put a partial 64-column step at the end of both lane loops."""
    for level in range(4):
        _report(f"dense L{level} P{P}", S.check_adapter_cells(_adapter, level, P, "dense", seed=10 + P))
    _report(f"dense tail P{P}", S.check_adapter_cells(_adapter, 0, P, "dense", E=1278, mid=98, seed=20 + P))


@pytest.mark.parametrize("name", S.GEOMETRY)
@pytest.mark.parametrize("level", range(4))
def test_adapter_splat_geometry_bit_exact(name, level):
    for coord_fp16 in (True, False):
        for scale in (1.0, 0.5, 3.0):
            _report(f"{name} L{level}", S.check_adapter_geometry(_adapter, name, level, coord_fp16, scale))


@pytest.mark.parametrize("level", range(4))
def test_adapter_fp16_coordinate_quantisation(level):
    for coord_fp16 in (True, False):
        for axis in (0, 1):
            _report(f"quant L{level}", S.check_adapter_quant(_adapter, level, coord_fp16, axis, scale=1.0 if axis else 3.0))


# ------------------------------------------------------------------------------------------------ time embedding
@pytest.mark.parametrize("t", [[999], [981, 1], [0, 1, 500, 981, 999, 21, 261, 741, 2]])
def test_time_embedding_per_element(t):
    m, sd = UC.get_model()
    _report(f"time B{len(t)}", S.check_time_embedding(m.time_embedding_rows, sd, m.cfg, t))


def test_time_embedding_rows_do_not_depend_on_the_batch():
    """Each row is computed on its own: row b of a B = 9 call equals a B = 1 call at that timestep bit for bit."""
    m, _ = UC.get_model()
    ts = [0.0, 1, 500, 981, 999, 21, 261, 741, 2]
    e9, p9 = m.time_embedding_rows(torch.tensor(ts))
    for j in (0, 3, 8):
        e1, p1 = m.time_embedding_rows(torch.tensor([ts[j]]))
        assert torch.equal(e1[0], e9[j]) and torch.equal(p1[0], p9[j]), ts[j]


# ------------------------------------------------------------------------------------------------ whole UNet, [B] t
_T = torch.tensor([981.0, 1.0])


def _unet_runs():
    """B = 2 at t = [981, 1]: the native output, the oracle's, the native output of the whole batch reversed (inputs and
    timesteps), of the timesteps alone reversed, and of each element alone at its timestep."""
    m, sd = UC.get_model()
    x = UC.randn((2, 4, 2, 8, 8), 2).half()
    ehs = UC.randn((2, 16, 77, 768), 3).half()
    with torch.no_grad():
        ref = O.unet_forward(sd, O.OracleConfig(), x.float(), _T, ehs.float(), None)

    def run(xx, t, ee):
        return m(xx.cuda(), t, ee.cuda(), return_dict=False)[0].float().cpu()

    out = run(x, _T.cuda(), ehs)
    reversed_batch = run(x.flip(0), _T.flip(0).cuda(), ehs.flip(0))
    t_reversed = run(x, _T.flip(0).cuda(), ehs)
    singles = [run(x[b:b + 1], float(_T[b]), ehs[b:b + 1]) for b in range(2)]
    torch.cuda.synchronize()
    return out, ref, reversed_batch, t_reversed, singles


def test_unet_batch_timesteps_per_element_and_frame():
    out, ref, reversed_batch, t_reversed, singles = _unet_runs()
    for b in range(2):
        for f in range(out.shape[2]):
            p = UC.psnr(out[b, :, f], ref[b, :, f])
            print(f"\nbatch {b} (t = {int(_T[b])}) frame {f}: {p:.1f} dB against the oracle")
            assert p >= 40.0, (b, f, p)
        # the batched forward equals the B = 1 forward at that timestep (GroupNorm float-atomics level)
        p1 = UC.psnr(out[b:b + 1], singles[b])
        print(f"batch {b}: {p1:.1f} dB against the B = 1 forward")
        assert p1 >= 60.0, (b, p1)
        # reversing the batch with its timesteps reverses the outputs ...
        ps = UC.psnr(reversed_batch[1 - b], out[b])
        assert ps >= 60.0, (b, ps)
        # ... and each element's timestep matters: the same element at the other timestep is far from it
        far = UC.psnr(t_reversed[b], out[b])
        print(f"batch {b}: {ps:.1f} dB reversed with its timestep, {far:.1f} dB at the other timestep")
        assert far < 50.0, (b, far)
