"""`python -m videoswap_b200.run` without a GPU: the shipped test configs parse into the dict the runner reads, the
dataset's frame selection, transforms and TAP slicing against restatements on synthetic frame directories, torchvision's
Resize / CenterCrop on PIL bit for bit, the file names save_video_to_dir writes, and every refusal raised before a model
is built."""
import copy
import glob
import json
import os

import numpy as np
import pytest
import torch
from PIL import Image

from tests.run_fixtures import SCHEDULER_CONFIG
from videoswap_b200 import data, formats, run

GOLD = os.path.join(os.path.dirname(__file__), "golden")
CONFIGS = sorted(glob.glob(os.path.join(GOLD, "test_videoswap", "*", "*.yml")))


def test_every_shipped_config_parses_into_the_runner_dict(tmp_path):
    assert len(CONFIGS) == 30
    for path in CONFIGS:
        opt = run.load_config(path)
        name = os.path.splitext(os.path.basename(path))[0]
        assert opt["name"] == name and opt["mixed_precision"] == "fp16" and opt["manual_seed"] == 74831, path
        # `!!float` gives floats, `~` gives None, YAML booleans stay booleans
        assert isinstance(opt["train"]["optimizer"]["lr"], float), path
        assert isinstance(opt["logger"]["save_checkpoint_freq"], float), path
        ds = opt["datasets"]
        assert ds["type"] == "SingleVideoPointDataset" and ds["num_frames"] == 16 and ds["total_frames"] in (48, 64, 96)
        assert isinstance(ds["prompt"], str) and isinstance(ds["path"], str), path
        assert [t["type"] for t in ds["video_transform"]][-2:] == ["ToTensor", "Normalize"], path
        assert len(data.build_transforms(ds["video_transform"])) == 1, path
        ec = opt["val"]["editing_config"]
        assert ec["use_invertion_latents"] is True and isinstance(ec["num_inference_steps"], int), path
        assert isinstance(ec["use_blend"], bool) and isinstance(ec["guidance_scale"], float), path
        for key, edit in ec["editing_prompts"].items():
            assert "->" in edit["replace"], (path, key)
            assert edit.get("tap_path") is None or isinstance(edit["tap_path"], str), (path, key)
            assert edit.get("select_point") is None or all(isinstance(s, str) for s in edit["select_point"]), (path, key)
            if edit.get("lora_path") is not None:
                assert len(edit["lora_path"].split("---")) == 2, (path, key)
        assert opt["val"]["save_type"] == "video"
        run.check_options(opt)
        # path.visualization: results/<name>/visualization under the root, unless given
        parsed = run.parse_options(copy.deepcopy(opt), root_path=str(tmp_path))
        assert parsed["path"]["visualization"] == os.path.join(str(tmp_path), "results", name, "visualization")
        given = copy.deepcopy(opt)
        given["path"]["visualization"] = "elsewhere"
        assert run.parse_options(given)["path"]["visualization"] == "elsewhere"


def test_select_frame_idx_matches_its_restatement():
    for end in (5, 16, 47, 48, 63, 64, 96, 100):
        for n in (2, 4, 8, 16):
            step = end // (n - 1)
            assert formats.select_frame_idx(0, end, n) == [i * step for i in range(n)], (end, n)


def _frames(d, n, w, h):
    d.mkdir(parents=True)
    g = torch.Generator().manual_seed(w * 7 + n)
    for i in range(n):
        arr = torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8).numpy()
        Image.fromarray(arr, "RGB").save(d / f"frame_{i:04d}.png")
    return d


def _tap(path, t, p, seed):
    g = torch.Generator().manual_seed(seed)
    tap = {"pred_tracks": torch.rand((t, p, 2), generator=g) * 300, "point_embedding": torch.randn((p, 1280), generator=g),
           "point_name2id": {f"pt{i}": i for i in range(p)}}
    torch.save(tap, path)
    return tap


@pytest.mark.parametrize("w,h", [(640, 360), (1280, 720)])
@pytest.mark.parametrize("transform,size", [
    ([{"type": "Resize", "size": 512}], lambda w, h: (int(512 * w / h), 512)),
    ([{"type": "Resize", "size": [448, 768]}], lambda w, h: (768, 448)),
    ([{"type": "Resize", "size": 512}, {"type": "CenterCrop", "size": 512}], lambda w, h: (512, 512)),
])
def test_dataset_selection_sizes_and_conditions(tmp_path, w, h, transform, size):
    frames = _frames(tmp_path / "frames", 64, w, h)
    tap = _tap(tmp_path / "TAP.pth", 64, 5, seed=w)
    opt = {"path": str(frames), "prompt": "a cat", "num_frames": 16, "total_frames": 48, "tap_path": str(tmp_path / "TAP.pth"),
           "video_transform": transform + [{"type": "ToTensor"}, {"type": "Normalize", "mean": [0.5], "std": [0.5]}]}
    ds = data.SingleVideoPointDataset(opt)
    select = [i * (48 // 15) for i in range(16)]
    assert ds.select_id == select
    assert ds.video == [frames / f"frame_{i:04d}.png" for i in select]
    W, H = size(w, h)
    assert (ds.size_x, ds.size_y) == (W, H)
    got = ds.get_frames()
    assert len(got) == 16 and all(f.mode == "RGB" and f.size == (W, H) for f in got)
    # the frames are the transforms applied to the selected files, in the config's order
    want = Image.open(ds.video[3]).convert("RGB")
    for t in data.build_transforms(transform):
        want = t(want)
    assert np.array_equal(np.asarray(got[3]), np.asarray(want))
    for cond in (ds.get_conditions(), ds.get_conditions(str(tmp_path / "TAP.pth"))):
        assert torch.equal(cond["pred_tracks"], tap["pred_tracks"][select])
        assert torch.equal(cond["point_embedding"], tap["point_embedding"])
        assert cond["point_name2id"] == tap["point_name2id"] and cond["img_size"] == (W, H)
    # a TAP file whose embedding rows do not match its points: the reference's assert, as a ValueError
    bad = dict(tap, point_embedding=tap["point_embedding"][:4])
    torch.save(bad, tmp_path / "bad.pth")
    with pytest.raises(ValueError, match="point_embedding"):
        ds.get_conditions(str(tmp_path / "bad.pth"))
    # no tap_path in the config: no source conditions
    no_tap = data.SingleVideoPointDataset({k: v for k, v in opt.items() if k != "tap_path"})
    assert no_tap.get_conditions() is None


def test_dataset_takes_fewer_frames_than_total(tmp_path):
    frames = _frames(tmp_path / "f", 20, 64, 48)
    ds = data.SingleVideoPointDataset({"path": str(frames), "prompt": "p", "num_frames": 4, "total_frames": 64,
                                       "video_transform": [{"type": "Resize", "size": 32}]})
    assert ds.select_id == [0, 6, 12, 18] and ds.get_frames()[0].size == (42, 32)


@pytest.mark.parametrize("w,h", [(640, 360), (1280, 720), (360, 640), (333, 517)])
def test_transforms_equal_torchvision_bit_for_bit(w, h):
    T = pytest.importorskip("torchvision.transforms")
    g = torch.Generator().manual_seed(w + h)
    img = Image.fromarray(torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8).numpy(), "RGB")
    cases = [(data.Resize(512), T.Resize(512)), (data.Resize([448, 768]), T.Resize([448, 768])),
             (data.Resize([512]), T.Resize([512])), (data.Resize(h), T.Resize(h)),
             (data.CenterCrop(256), T.CenterCrop(256)), (data.CenterCrop([200, 301]), T.CenterCrop([200, 301])),
             (data.CenterCrop([h + 3, w - 7]), T.CenterCrop([h + 3, w - 7])),       # padded along one side
             (data.CenterCrop(max(w, h) + 10), T.CenterCrop(max(w, h) + 10))]
    for mine, theirs in cases:
        a, b = mine(img), theirs(img)
        assert a.size == b.size and a.mode == b.mode, (mine, a.size, b.size)
        assert np.array_equal(np.asarray(a), np.asarray(b)), mine


def _video(n=3, size=(32, 24)):
    return [Image.new("RGB", size, (40 * i, 100, 200)) for i in range(n)]


def test_save_video_to_dir_file_names(tmp_path, monkeypatch):
    run.save_video_to_dir(_video(), str(tmp_path / "a"), "edit", save_type="frame")
    assert sorted(os.listdir(tmp_path / "a" / "frames")) == ["00000_edit.jpg", "00001_edit.jpg", "00002_edit.jpg"]
    assert os.listdir(tmp_path / "a") == ["frames"]
    run.save_video_to_dir(_video(), str(tmp_path / "b"), "edit", save_type="gif", fps=4)
    assert os.listdir(tmp_path / "b") == ["edit.gif"]
    with Image.open(tmp_path / "b" / "edit.gif") as gif:
        assert gif.n_frames == 3 and gif.info["duration"] == 250 and gif.info["loop"] == 0
    run.save_video_to_dir(_video(), str(tmp_path / "c"), "edit", save_type="frame_gif")
    assert sorted(os.listdir(tmp_path / "c")) == ["edit.gif", "frames"]
    assert len(os.listdir(tmp_path / "c" / "frames")) == 3
    # video: mp4 through imageio; without it a clear ImportError, before anything is written
    import builtins
    real_import = builtins.__import__

    def no_imageio(name, *a, **k):
        if name == "imageio" or name.startswith("imageio."):
            raise ImportError("No module named 'imageio'")
        return real_import(name, *a, **k)
    monkeypatch.setattr(builtins, "__import__", no_imageio)
    for save_type in ("video", "frame_video"):
        with pytest.raises(ImportError, match="imageio"):
            run.save_video_to_dir(_video(), str(tmp_path / save_type), "edit", save_type=save_type)
        assert not os.path.exists(tmp_path / save_type)


def test_save_results_layout_and_suffixes(tmp_path):
    results = {"to_dog": _video(), "to_dog_vispoint": _video()}
    opt = {"name": "cfg", "path": {"visualization": str(tmp_path / "v")}, "val": {"save_type": "frame_gif"}}
    last = run.save_results(opt, _video(), results)
    assert last == str(tmp_path / "v" / "to_dog_vispoint")
    assert sorted(os.listdir(tmp_path / "v")) == ["source", "to_dog", "to_dog_vispoint"]
    assert sorted(os.listdir(tmp_path / "v" / "to_dog")) == ["frames", "to_dog.gif"]
    assert sorted(os.listdir(tmp_path / "v" / "source" / "frames"))[0] == "00000_source.jpg"
    # use_suffix; and without 'frame' every edit goes into the visualization directory itself
    opt = {"name": "cfg", "path": {"visualization": str(tmp_path / "w")}, "val": {"save_type": "gif", "use_suffix": True}}
    assert run.save_results(opt, _video(), results) == str(tmp_path / "w")
    assert sorted(os.listdir(tmp_path / "w")) == ["source", "to_dog_cfg.gif", "to_dog_vispoint_cfg.gif"]
    assert os.listdir(tmp_path / "w" / "source") == ["source.gif"]


def test_scheduler_config_overrides_and_defaults():
    assert run.scheduler_kwargs(SCHEDULER_CONFIG) == {
        "beta_end": 0.012, "beta_schedule": "scaled_linear", "beta_start": 0.00085, "num_train_timesteps": 1000,
        "set_alpha_to_one": False, "steps_offset": 1}
    # the reference's overrides: steps_offset -> 1, clip_sample -> False
    with pytest.warns(UserWarning, match="steps_offset"):
        k = run.scheduler_kwargs(dict(SCHEDULER_CONFIG, steps_offset=0, clip_sample=True))
    assert k["steps_offset"] == 1
    # keys left out take diffusers' DDIMScheduler defaults
    with pytest.warns(UserWarning):
        k = run.scheduler_kwargs({"set_alpha_to_one": False})
    assert (k["beta_start"], k["beta_end"], k["beta_schedule"]) == (0.0001, 0.02, "linear")


def _config(tmp_path, **over):
    """A config whose pretrained directory holds only scheduler/scheduler_config.json: enough to reach every refusal."""
    sd = tmp_path / "sd" / "scheduler"
    sd.mkdir(parents=True, exist_ok=True)
    (sd / "scheduler_config.json").write_text(json.dumps(dict(SCHEDULER_CONFIG, **over.pop("scheduler", {}))))
    opt = run.load_config(CONFIGS[0])
    opt["path"]["pretrained_model_path"] = str(tmp_path / "sd")
    opt["path"]["visualization"] = str(tmp_path / "vis")
    opt["val"]["save_type"] = "frame_gif"
    for path, value in over.items():
        node = opt
        keys = path.split("/")
        for k in keys[:-1]:
            node = node[k]
        node[keys[-1]] = value
    return opt


@pytest.mark.parametrize("over,err,match", [
    ({"models/unet/type": "UNet3DConditionModel"}, NotImplementedError, "unet type"),
    ({"models/adapter/type": "T2IAdapter"}, NotImplementedError, "adapter type"),
    ({"datasets/video_transform": [{"type": "RandomCrop", "size": 256}]}, NotImplementedError, "RandomCrop"),
    ({"mixed_precision": "bf16"}, ValueError, "fp16"),
    ({"mixed_precision": "no"}, ValueError, "fp16"),
    ({"scheduler": {"prediction_type": "v_prediction"}}, ValueError, "prediction_type"),
    ({"scheduler": {"timestep_spacing": "trailing"}}, ValueError, "timestep_spacing"),
    ({"scheduler": {"thresholding": True}}, ValueError, "thresholding"),
    ({"scheduler": {"beta_schedule": "squaredcos_cap_v2"}}, ValueError, "beta_schedule"),
    ({"scheduler": {"set_alpha_to_one": True}}, ValueError, "set_alpha_to_one"),
    ({"scheduler": {"trained_betas": [0.1] * 1000}}, ValueError, "trained_betas"),
])
def test_refusals_come_before_any_model(tmp_path, monkeypatch, over, err, match):
    def built(*a, **k):
        raise AssertionError("a model was built before the refusal")
    monkeypatch.setattr(run, "load_pipeline", built)
    monkeypatch.setattr(run, "SingleVideoPointDataset", built)
    opt = _config(tmp_path, **over)
    before = copy.deepcopy(opt)
    with pytest.raises(err, match=match):
        run.run_config(opt)
    assert opt == before                                  # the caller's dict is not changed
    assert not os.path.exists(tmp_path / "vis")


def test_video_without_imageio_is_refused_before_any_model(tmp_path, monkeypatch):
    import builtins
    real_import = builtins.__import__

    def no_imageio(name, *a, **k):
        if name == "imageio":
            raise ImportError("No module named 'imageio'")
        return real_import(name, *a, **k)
    monkeypatch.setattr(builtins, "__import__", no_imageio)
    monkeypatch.setattr(run, "load_pipeline", lambda *a, **k: pytest.fail("a model was built"))
    opt = _config(tmp_path)
    opt["val"]["save_type"] = "video"
    with pytest.raises(ImportError, match="imageio"):
        run.run_config(opt)


def test_seed_and_order_up_to_the_models(tmp_path, monkeypatch):
    """A config without manual_seed draws one as test.py does; the models are loaded after seeding, the dataset after
    the models, and the random state at the end is the seed's."""
    calls = []

    class Stop(Exception):
        pass

    def fake_pipeline(opt, sched, tokenizer=None):
        calls.append(("pipeline", opt["manual_seed"], sched, tokenizer))
        return "pipe"

    def fake_dataset(opt):
        calls.append(("dataset", opt["path"]))
        raise Stop
    monkeypatch.setattr(run, "load_pipeline", fake_pipeline)
    monkeypatch.setattr(run, "SingleVideoPointDataset", fake_dataset)
    opt = _config(tmp_path, manual_seed=1234)
    with pytest.raises(Stop):
        run.run_config(opt, tokenizer="tok")
    assert calls[0][:2] == ("pipeline", 1234) and calls[0][3] == "tok" and calls[1][0] == "dataset"
    assert calls[0][2]["beta_schedule"] == "scaled_linear"
    import random
    drawn = (torch.rand(3), np.random.rand(3), random.random())
    torch.manual_seed(1234)
    np.random.seed(1234)
    random.seed(1234)
    assert torch.equal(drawn[0], torch.rand(3)) and np.array_equal(drawn[1], np.random.rand(3))
    assert drawn[2] == random.random()
    opt = _config(tmp_path, manual_seed=None)
    with pytest.raises(Stop):
        run.run_config(opt)
    assert 1 <= calls[2][1] <= 10000


def test_main_parses_the_command_line(tmp_path, monkeypatch):
    seen = {}
    monkeypatch.setattr(run, "run_config", lambda opt: seen.setdefault("opt", opt) and "out")
    assert run.main(["-opt", CONFIGS[0]]) == "out"
    assert seen["opt"] == run.load_config(CONFIGS[0])


def test_runner_imports_none_of_the_reference_dependencies():
    import subprocess
    import sys
    code = ("import sys, videoswap_b200.run, videoswap_b200.data; "
            "print(sorted(m for m in ('diffusers', 'omegaconf', 'accelerate', 'torchvision', 'imageio') if m in sys.modules))")
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, check=True,
                         cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    assert out.stdout.strip() == "[]"
