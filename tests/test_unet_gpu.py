"""GPU parity tests (pytest -m gpu) of the whole path through the reference-facing surface:
AnimateDiffUNet3DModel.forward / VideoSwapPipeline loop body / SparsePointAdapter vs the CPU oracle and vs the
fixtures generated from the reference's own files.  Tolerance (north_star): PSNR >= 40 dB in fp16."""
import pytest
import torch

from tests import unet_checks as U

pytestmark = pytest.mark.gpu
PSNR_MIN = 40.0


@pytest.mark.parametrize("name", ["full_arch_small", "full_arch_c1"])
def test_unet_matches_reference_golden(name):
    """full_arch_c1 = BASELINE configs[0] at its real size ([1,4,1,64,64], N = 4096 attention) from the reference's files."""
    r = U.unet_vs_reference_golden(name)
    assert r["psnr"] >= PSNR_MIN, r


@pytest.mark.parametrize("kw", [dict(B=1, Fr=2, hw=8, edlora=True), dict(B=2, Fr=3, hw=16, edlora=True, residuals=True),
                                dict(B=1, Fr=16, hw=8, edlora=False, t=1),
                                dict(B=1, Fr=2, hw=8, w=24, edlora=True, residuals=True),    # non-square (56x96-like aspect)
                                dict(B=1, Fr=1, hw=8, edlora=True),                          # C1: single frame
                                dict(B=1, Fr=24, hw=8, edlora=False),                        # longest clip of the PE table
                                dict(B=1, Fr=1, hw=64, edlora=True),                         # C1 at its real 64x64 latent
                                dict(B=1, Fr=4, hw=64, edlora=True, residuals=True, taps=True),   # headline resolution, 4 frames
                                dict(B=2, Fr=2, hw=64, w=32, edlora=True, residuals=True)])  # CFG batch, 512x256
def test_unet_matches_oracle(kw):
    r = U.unet_vs_oracle(**kw)
    assert r["finite"] and r["psnr"] >= PSNR_MIN, r
    for name, tp in r.get("taps", {}).items():          # every block output, not only the final 4-channel epsilon
        assert tp["psnr"] >= PSNR_MIN, (name, tp)


def test_fp32_latents_take_the_same_path():
    """The reference keeps latents in the scheduler's dtype; fp32 in -> fp32 out, same kernels (io_f32 = 1)."""
    m, _ = U.get_model()
    x = U.randn((1, 4, 2, 8, 8), 41)
    e = U.randn((1, 77, 768), 42).half().cuda()
    o16 = m(x.half().cuda(), 501, e, return_dict=False)[0]
    o32 = m(x.half().float().cuda(), 501, e, return_dict=False)[0]
    assert o32.dtype == torch.float32 and o16.dtype == torch.float16
    assert U.psnr(o32, o16.float().cpu()) >= 60.0


def test_frame_count_beyond_pe_table_raises():
    m, _ = U.get_model()
    x = torch.zeros(1, 4, 25, 8, 8, dtype=torch.float16, device="cuda")
    with pytest.raises(Exception):
        m(x, 1, torch.zeros(1, 77, 768, dtype=torch.float16, device="cuda"))


def test_residual_list_is_consumed_in_place():
    m, _ = U.get_model()
    x = torch.zeros(1, 4, 1, 8, 8, dtype=torch.float16, device="cuda")
    res = [torch.zeros(1, c, max(8 >> l, 1), max(8 >> l, 1), dtype=torch.float16, device="cuda")
           for l, c in enumerate(m.cfg.block_out_channels)]
    m(x, 1, torch.zeros(1, 77, 768, dtype=torch.float16, device="cuda"), down_block_additional_residuals=res)
    assert len(res) == 0          # the reference pops the list (unet.py:422,435)


def test_denoise_loop_matches_oracle():
    r = U.pipeline_vs_oracle(steps=3)
    assert r["psnr"] >= PSNR_MIN, r


def test_pipeline_call_with_conditions_matches_oracle():
    """VideoSwapPipeline.__call__: adapter from `conditions`, t2i window (closed after iteration 0), CFG, DDIM, and the
    reference's final 'b c f h w -> (b f) c h w' (pipeline_videoswap.py:525-610)."""
    r = U.pipeline_call_vs_oracle(iters=3)
    assert r["shape"] == r["ref_shape"] == (2, 4, 16, 16), r
    assert r["psnr"] >= PSNR_MIN, r
    assert r["psnr_if_window_ignored"] < r["psnr"] - 10.0, r     # the window really closed after iteration 0 ...
    assert r["psnr_if_never_applied"] < r["psnr"] - 10.0, r      # ... and was open in iteration 0


@pytest.mark.parametrize("convention", ["0.19.3", "0.21"])
def test_invert_matches_oracle(convention):
    r = U.invert_vs_oracle(iters=3, convention=convention)
    assert r["psnr"] >= PSNR_MIN, r


def test_workspace_survives_other_shapes_under_a_captured_graph():
    """ADVICE r1: a captured graph holds raw pointers into the workspace.  Smaller shapes re-use the arena (the replay stays
    correct); a LARGER shape must fail loudly instead of re-allocating under the graph."""
    from videoswap_b200 import DDIMScheduler, VideoSwapPipeline
    from videoswap_b200.pipeline import GraphedStep
    m = U.fresh_model()                        # own handle: its arena has only ever seen the shapes of this test
    pipe = VideoSwapPipeline(m, DDIMScheduler())
    pipe.scheduler.set_timesteps(50)
    lat = U.randn((1, 4, 2, 16, 16), 33).half().cuda()
    emb = U.randn((2, 16, 77, 768), 34).half().cuda()
    g = GraphedStep(pipe, lat, emb, 7.5)
    ref = g(lat, 981).clone()
    small = m(torch.zeros(1, 4, 1, 8, 8, dtype=torch.float16, device="cuda"), 1, emb[:1], return_dict=False)[0]   # B=1 inversion-like
    assert torch.isfinite(small).all()
    again = g(lat, 981).clone()
    torch.cuda.synchronize()
    assert U.psnr(again, ref) >= 60.0
    with pytest.raises(Exception, match="pinned"):
        m(torch.zeros(2, 4, 4, 32, 32, dtype=torch.float16, device="cuda"), 1, emb, return_dict=False)
    del g
    big = m(torch.zeros(2, 4, 4, 32, 32, dtype=torch.float16, device="cuda"), 1, emb, return_dict=False)[0]       # unpinned: grows
    assert torch.isfinite(big).all()


def test_cuda_graph_step_equals_eager_step():
    from videoswap_b200 import DDIMScheduler, VideoSwapPipeline
    from videoswap_b200.pipeline import GraphedStep
    m, _ = U.get_model()
    pipe = VideoSwapPipeline(m, DDIMScheduler())
    pipe.scheduler.set_timesteps(50)
    lat = U.randn((1, 4, 2, 8, 8), 31).half().cuda()
    emb = U.randn((2, 16, 77, 768), 32).half().cuda()
    g = GraphedStep(pipe, lat, emb, 7.5)
    for t in (981, 501, 1):                      # one captured graph, replayed at different timesteps
        ref = pipe.step(lat, t, emb, 7.5)
        out = g(lat, t).clone()
        torch.cuda.synchronize()
        assert torch.isfinite(out).all()
        # same kernels, same inputs: only fp32-atomic summation order in the GroupNorm statistics may differ
        assert U.psnr(out, ref) >= 60.0, (t, U.psnr(out, ref))


def test_adapter_fp16_coordinates_match_reference_golden():
    """Product default path: fp16 coordinate quantisation (SURVEY P7) against the reference's half-precision adapter."""
    r = U.adapter_fp16_vs_golden()
    assert all(r["same_support"]), r
    for e, ref in zip(r["errs"], r["refs"]):
        assert e <= 2 ** -7 * ref + 4e-3, r       # fp16 accumulation order differs (gather vs the reference's += sequence)


def test_adapter_matches_reference_golden():
    r = U.adapter_vs_golden()
    for e, ref in zip(r["errs"], r["refs"]):
        assert e <= 2 ** -8 * ref + 2e-3, r


# ---------------------------------------------------------------------------------------------------- attention controllers
def test_explicit_probability_attention():
    from tests import p2p_checks as P
    for kw in (dict(B=3, N=256, C=1280), dict(B=4, N=64, C=1280, seed=171), dict(B=4, N=256, NK=77, C=1280, kv_div=2, seed=172),
               dict(B=2, N=200, NK=77, C=640, seed=173), dict(B=2, N=100, C=320, seed=174)):
        r = P.explicit_attention_check(**kw)
        assert r["probs"]["ok"] and r["out"]["ok"], (kw, r)
        assert r["row_sum_err"] <= 4e-3 and r["out_err"] <= 2 ** -8 * r["out_ref"] + 2e-3, (kw, r)


def test_attention_hook_delivers_the_reference_maps():
    """register_attention_control + forward: the 16x16 / 8x8 layers (below 32^2 queries) hand [(b f), 8, s, t] to the
    controller in the reference's order (down 2 x (self, cross), mid, up 3 x ...), and an in-place edit reaches epsilon."""
    from tests import p2p_checks as P
    r = P.unet_hook_vs_oracle(Fr=2, hw=64 // 2)           # 32x32 latent: levels 32^2 (not controlled), 16^2, 8^2, 4^2
    assert r["registered"] == 32, r
    assert r["min_map_psnr"] >= PSNR_MIN and r["eps_psnr"] >= PSNR_MIN, r
    e = P.unet_hook_vs_oracle(Fr=2, hw=16, edit=True)
    assert e["min_map_psnr"] >= PSNR_MIN and e["eps_psnr"] >= PSNR_MIN, e


@pytest.mark.parametrize("kind", ["refine", "replace"])
def test_device_controllers_match_the_reference_classes(kind):
    """Store -> refine / replace of the cross maps, masked self-attention replacement, blend mask and latent blend, replayed
    against the fixture the reference's own classes produced (oracle/make_golden_p2p.py)."""
    from tests import p2p_checks as P
    r = P.replay_vs_reference_fixture(kind)
    assert r["n_masks"][0] == r["n_masks"][1]
    assert r["map_err"] <= 2e-3 and r["latent_err"] <= 4e-3, r
    assert r["mask_mismatch"] <= 0.01 * r["mask_pixels"], r      # thresholded masks: fp16 maps vs the fp32 reference


def test_use_blend_flow_matches_oracle():
    """Inversion with the store registered, then the editing loop with cross refine + masked self replacement + latent blend
    (the `use_blend: true` body of the shipped configs at 512x512, 2 + 2 steps) through pipe.invert / pipe(..., controller=)."""
    from tests import p2p_checks as P
    r = P.edit_flow_vs_oracle(n_steps=2)
    assert r["steps"] == (2, 2) and r["stored_maps"] == 12, r
    assert r["inversion_psnr"] >= PSNR_MIN and r["edit_psnr"] >= PSNR_MIN, r
    assert 0.05 < r["mask_fill"] < 0.95, r                               # the blend really mixes source and target latents
    assert r["unused_forced"] == (0, 0) and r["masks_checked"][1] == 2, r # both sides computed the same number of masks
    assert r["mask_mismatch"] <= 0.03 * r["mask_pixels"], r              # thresholded maps: fp16 device maps vs fp32 oracle


def test_edlora_merge_in_place_and_restore():
    """SURVEY 8f-4 (ED-LoRA file -> UNet weights, convert_edlora_to_diffusers.py:36-96): the in-place merge reaches the kernels
    (lazy re-pack), matches the oracle on independently merged weights, and restore brings back the parameters bit-exactly."""
    r = U.edlora_merge_vs_oracle()
    assert r["pairs"] == r["touched"] > 20, r
    assert r["psnr"] >= 40.0 and r["psnr_unmerged_vs_merged_ref"] < r["psnr"] - 15.0, r      # the merge really changed the output
    assert r["restored_params_bit_exact"] and r["psnr_restored_vs_before"] >= 60.0, r
