"""`VideoSwapPipeline.validation` on an editing_config with `use_blend`, against the same flow composed by hand from the
pipeline's public calls: `invert` with an AttentionStore, edit controllers built from the tensors the reference's own
make_controller produced (tests/golden/controllers.pt), `pipe(...)` with them, and the ED-LoRA merge and restore.

Seeded full-size UNet, VAE, text encoder and adapter; oracle/chunk_tokenizer.py as the tokenizer; 2 frames of 256 x 256,
4 DDIM steps, two edits: one with an ED-LoRA file and `select_point`, one without a LoRA and with `tap_path`.  256 x 256
(32 x 32 latents) is the smallest size at which every map the latent blend reads (down_cross[2:4], up_cross[:3]) has one
resolution, which the reference's SpatialBlender needs as well.

GroupNorm sums its statistics with float atomics, so two runs of one flow agree to the last bits only.  The bar is therefore
the run-to-run envelope: the composition runs twice, and validation must agree with both runs at least as closely as they
agree with each other, minus 3 dB (the envelope capped at 50 dB, where 8-bit frames differ by rounding only)."""
import copy
import math

import numpy as np
import pytest
import torch

import videoswap_b200 as V
from oracle import make_golden_controllers as M
from oracle.chunk_tokenizer import ChunkTokenizer
from tests import unet_checks as U
from tests.test_controllers_cpu import GOLD, _assert_equal
from videoswap_b200 import formats, p2p

pytestmark = pytest.mark.gpu

STEPS, FRAMES, SIZE = 4, 2, 256
SOURCE = "a kitten playing with a ball of yarn"
EDIT_LORA = {"row": "refine_edlora", "replace": "kitten -> <catA1> <catA2>"}
EDIT_TAP = {"row": "refine_insert_split_words", "replace": "kitten -> small puppy"}
NAMES = ["head", "tail", "paw", "ear", "nose", "back"]


def _row(name):
    return next(r for r in M.ROWS if r["name"] == name)


def _blend_cfg(row):
    return {"cross_replace_steps": row["cross"], "self_replace_steps": row["self_"], "blend_th": row["th"][0]}


def _tracks(seed, P=len(NAMES)):
    g = torch.Generator().manual_seed(seed)
    t = torch.rand((FRAMES, P, 2), generator=g) * (SIZE - 20) + 10
    t[0, 1] = -1.0                                  # invisible in frame 0
    return t


@pytest.fixture(scope="module")
def setup(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("validation")
    unet, sd = U.get_model()
    g = torch.Generator().manual_seed(401)
    lora_unet = {}
    for k, w in sd.items():
        dn = formats.lora_down_name(k)
        if dn == k or "motion_modules" in k or not any(s in k for s in ("down_blocks.1.", "up_blocks.2.attentions.0.")):
            continue
        down, up = 0.05 * torch.randn((4, w.shape[1]), generator=g), 0.05 * torch.randn((w.shape[0], 4), generator=g)
        if w.dim() == 4:
            down, up = down[:, :, None, None], up[:, :, None, None]
        lora_unet[dn], lora_unet[dn.replace("lora_down", "lora_up")] = down, up
    lora_te = {}
    for i in (0, 6, 11):
        for site, (o, n) in (("self_attn.q_proj", (768, 768)), ("mlp.fc1", (3072, 768))):
            lora_te[f"text_model.encoder.layers.{i}.{site}.lora_down.weight"] = 0.05 * torch.randn(4, n, generator=g)
            lora_te[f"text_model.encoder.layers.{i}.{site}.lora_up.weight"] = 0.05 * torch.randn(o, 4, generator=g)
    concepts = {c: 0.02 * torch.randn(16, 768, generator=g) for c in ("<catA1>", "<catA2>")}
    lora_path = tmp / "edlora_catA.pth"
    torch.save({"params": {"new_concept_embedding": concepts, "unet": lora_unet, "text_encoder": lora_te}}, lora_path)
    tap_path = tmp / "TAP_puppy.pth"
    torch.save({"pred_tracks": _tracks(403), "point_embedding": torch.randn((len(NAMES), 1280), generator=g),
                "point_name2id": {n: i for i, n in enumerate(NAMES)}}, tap_path)
    source_conditions = {"pred_tracks": _tracks(402), "point_embedding": torch.randn((len(NAMES), 1280), generator=g),
                         "point_name2id": {n: i for i, n in enumerate(NAMES)}, "img_size": (SIZE, SIZE), "index_list": None}
    from PIL import Image
    frames = [Image.fromarray(torch.randint(0, 256, (SIZE, SIZE, 3), generator=g, dtype=torch.uint8).numpy(), "RGB")
              for _ in range(FRAMES)]
    te = V.CLIPTextModel()
    pipe = V.VideoSwapPipeline(unet, V.DDIMScheduler(), adapter=V.SparsePointAdapter().half().cuda(),
                               inverse_scheduler=V.DDIMInverseScheduler(), vae=V.AutoencoderKL(), text_encoder=te,
                               tokenizer=ChunkTokenizer(base_vocab=te.get_input_embeddings().weight.shape[0]))

    class Dataset:
        def get_conditions(self, path):
            return formats.load_tap(path, img_size=(SIZE, SIZE))

    config = {
        "use_invertion_latents": True, "use_blend": True, "guidance_scale": 7.5, "visualize_point": True,
        "num_inference_steps": STEPS, "negative_prompt": "low quality", "t2i_guidance_scale": 0.5, "t2i_start": 0.0,
        "t2i_end": 0.5,
        "editing_prompts": {
            "to_catA": {"replace": EDIT_LORA["replace"], "lora_path": f"{lora_path}---0.7", "select_point": ["tail", "head"],
                        "blend_cfg": _blend_cfg(_row(EDIT_LORA["row"]))},
            "to_puppy": {"replace": EDIT_TAP["replace"], "tap_path": str(tap_path), "select_point": None, "guidance_scale": 5.0,
                         "negative_prompt": "blurry", "blend_cfg": _blend_cfg(_row(EDIT_TAP["row"]))},
        },
    }
    return dict(pipe=pipe, frames=frames, cond=source_conditions, config=config, dataset=Dataset(), lora_path=str(lora_path),
                tap_path=str(tap_path))


def _controller_from_fixture(row, store):
    """The controller from_reference makes of the reference's make_controller output, from the fixture's tensors."""
    fx = GOLD[row["name"]]

    def blender(b):
        nb = p2p.SpatialBlender(b["alpha_layers"], th=tuple(b["th"].tolist()), NUM_DDIM_STEPS=row["steps"],
                                prompt_choose="both" if bool(b["choose_both"]) else "source")
        nb.start_blend, nb.end_blend = (int(v) for v in b["start_end"])
        return nb
    ctl = p2p.AttentionRefine(fx["mapper"].cuda(), fx["alphas"].cuda(), num_steps=row["steps"],
                              cross_replace_alpha=fx["cross_replace_alpha"].cuda(), self_replace_steps=0.0,
                              latent_blend=blender(fx["latent_blend"]), additional_attention_store=store,
                              attention_blend=blender(fx["attention_blend"]), image_height=SIZE, image_width=SIZE)
    ctl.num_self_replace = tuple(fx["num_self_replace"].tolist())
    return ctl


def _composed(s):
    """validation's flow, written out with the pipeline's public calls."""
    pipe = s["pipe"]
    torch.manual_seed(0)
    store = p2p.AttentionStore()
    store.LOW_RESOURCE = True
    p2p.register_attention_control(pipe, store)
    inv = pipe.invert(prompt=SOURCE, video=s["frames"], num_inference_steps=STEPS, controller=store).latents.half()
    p2p.register_attention_control(pipe, None)
    out = {}
    # edit 1: ED-LoRA, select_point
    lora = formats.load_edlora(s["lora_path"])
    concept_cfg = formats.load_new_concept(pipe.tokenizer, pipe.text_encoder, lora["new_concept_embedding"])
    ub = formats.merge_edlora_into_unet(pipe.unet, lora["unet"], 0.7)
    tb = formats.merge_edlora_into_text_encoder(pipe.text_encoder, lora["text_encoder"], 0.7)
    pipe.set_new_concept_cfg(concept_cfg)
    ctl = _controller_from_fixture(_row(EDIT_LORA["row"]), store)
    p2p.register_attention_control(pipe, ctl)
    cond = copy.deepcopy(s["cond"])
    cond["index_list"] = [1, 0]
    out["to_catA"] = pipe(prompt=_row(EDIT_LORA["row"])["prompts"][1], negative_prompt="low quality", conditions=cond,
                          latents=inv, num_inference_steps=STEPS, guidance_scale=7.5, t2i_guidance_scale=0.5, t2i_start=0.0,
                          t2i_end=0.5, controller=ctl, output_type="pil").videos
    p2p.register_attention_control(pipe, None)
    formats.restore_unet(pipe.unet, ub)
    formats.restore_text_encoder(pipe.text_encoder, tb)
    pipe.set_new_concept_cfg(None)
    # edit 2: no LoRA, tap_path
    ctl = _controller_from_fixture(_row(EDIT_TAP["row"]), store)
    p2p.register_attention_control(pipe, ctl)
    out["to_puppy"] = pipe(prompt=_row(EDIT_TAP["row"])["prompts"][1], negative_prompt="blurry",
                           conditions=formats.load_tap(s["tap_path"], img_size=(SIZE, SIZE)), latents=inv,
                           num_inference_steps=STEPS, guidance_scale=5.0, t2i_guidance_scale=0.5, t2i_start=0.0, t2i_end=0.5,
                           controller=ctl, output_type="pil").videos
    p2p.register_attention_control(pipe, None)
    return out


def _arr(frames):
    return np.stack([np.asarray(f, dtype=np.float64) for f in frames])


def _psnr(a, b):
    mse = float(((_arr(a) - _arr(b)) ** 2).mean())
    return math.inf if mse == 0 else 10 * math.log10(255.0 ** 2 / mse)


def test_validation_equals_the_composed_flow(setup, monkeypatch):
    s = setup
    pipe = s["pipe"]
    te_rows = pipe.text_encoder.get_input_embeddings().weight.shape[0]
    unet_before = {k: p.detach().clone() for k, p in pipe.unet.named_parameters()}
    te_before = {k: p.detach().clone() for k, p in pipe.text_encoder.named_parameters()}

    built = []
    real = p2p.make_controller

    def recording(*a, **k):
        built.append(real(*a, **k))
        return built[-1]
    monkeypatch.setattr(p2p, "make_controller", recording)
    torch.manual_seed(0)
    res = pipe.validation(s["frames"], s["cond"], SOURCE, s["config"], train_dataset=s["dataset"])
    monkeypatch.setattr(p2p, "make_controller", real)
    torch.cuda.synchronize()

    assert sorted(res) == ["to_catA", "to_catA_vispoint", "to_puppy", "to_puppy_vispoint"]
    assert all(len(res[k]) == FRAMES and res[k][0].size == (SIZE, SIZE) for k in res)
    # the controllers validation built are the reference's, and they ran every step
    for ctl, edit in zip(built, (EDIT_LORA, EDIT_TAP)):
        _assert_equal(M.native_attributes(ctl), GOLD[edit["row"]], edit["row"])
        assert ctl.cur_step == STEPS and len(ctl.latent_blend.mask_list) == STEPS
    # nothing of the edits is left in the models: every parameter as before (the token embedding keeps the concept rows)
    assert pipe.new_concept_cfg is None
    for k, p in pipe.unet.named_parameters():
        assert torch.equal(p, unet_before[k]), k
    for k, p in pipe.text_encoder.named_parameters():
        if p.shape != te_before[k].shape:
            assert p.shape[0] == te_rows + 32 and torch.equal(p[:te_rows], te_before[k]), k
        else:
            assert torch.equal(p, te_before[k]), k

    a = _composed(s)
    b = _composed(s)
    torch.cuda.synchronize()
    for key in ("to_catA", "to_puppy"):
        env = min(_psnr(a[key], b[key]), 50.0)
        got = min(_psnr(res[key], a[key]), _psnr(res[key], b[key]))
        print(f"\n{key}: validation vs composition {got:.1f} dB, composition vs itself {_psnr(a[key], b[key]):.1f} dB")
        assert got >= env - 3.0, key
    # the two edits differ from each other (the prompts, the LoRA and the conditions reach the output)
    assert _psnr(res["to_catA"], res["to_puppy"]) < 30.0


def test_vispoint_frames_differ_only_inside_the_discs(setup):
    s = setup
    cfg = copy.deepcopy(s["config"])
    cfg["editing_prompts"] = {"to_puppy": cfg["editing_prompts"]["to_puppy"]}
    cfg["editing_prompts"]["to_puppy"]["select_point"] = ["tail", "nose"]
    res = s["pipe"].validation(s["frames"], s["cond"], SOURCE, cfg, train_dataset=s["dataset"])
    plain, drawn = _arr(res["to_puppy"]), _arr(res["to_puppy_vispoint"])
    tracks = formats.load_tap(s["tap_path"])["pred_tracks"]
    yy, xx = np.mgrid[0:SIZE, 0:SIZE]
    for f in range(FRAMES):
        inside = np.zeros((SIZE, SIZE), dtype=bool)
        for p in (NAMES.index("tail"), NAMES.index("nose")):
            x, y = (float(v) for v in tracks[f, p])
            if x >= 0 and y >= 0:
                inside |= (xx - x) ** 2 + (yy - y) ** 2 <= 6.5 ** 2
        changed = (plain[f] != drawn[f]).any(-1)
        assert changed.any() and not (changed & ~inside).any(), f
        assert (drawn[f][changed] == (0, 255, 0)).all()


def test_validation_refuses_what_it_cannot_run(setup):
    s = setup
    pipe = s["pipe"]
    for flag, err, match in (("use_invertion_latents", ValueError, "use_invertion_latents"),
                             ("visualize_attention", NotImplementedError, "show_cross_attention")):
        cfg = dict(s["config"], **{flag: flag == "visualize_attention"})
        with pytest.raises(err, match=match):
            pipe.validation(s["frames"], s["cond"], SOURCE, cfg)
    bare = V.VideoSwapPipeline(pipe.unet, text_encoder=pipe.text_encoder)
    with pytest.raises(ValueError, match="vae, tokenizer"):
        bare.validation(s["frames"], s["cond"], SOURCE, s["config"])
