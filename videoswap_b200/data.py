"""The reference's test-time dataset (videoswap/data/frame_point_dataset.py `SingleVideoPointDataset`, data/transform.py)
without torchvision: the source frames of a config's `datasets` entry as RGB PIL images, and the TAP conditions sliced to
the selected frames.  Host work only (file decoding and resizing of a few frames, once per run)."""
from __future__ import annotations

from pathlib import Path
from typing import Dict, List, Mapping, Optional, Sequence, Union

from . import formats

# transform types a config may list; ToTensor and Normalize only matter for training batches and are skipped by
# get_frames, as the reference's get_frames skips them
_TENSOR_TRANSFORMS = ("ToTensor", "Normalize")


class Resize:
    """torchvision.transforms.Resize on a PIL image, bilinear: an int (or a one-element list) is the new length of the
    shorter side, the longer one becomes int(size * long / short); a pair is (height, width).  An image already at the
    target size is returned as is, as torchvision returns it."""

    def __init__(self, size: Union[int, Sequence[int]]):
        if isinstance(size, int):
            size = [size]
        if len(size) not in (1, 2):
            raise ValueError(f"Resize size must be an int or a list of 1 or 2 ints, got {size!r}")
        self.size = [int(s) for s in size]

    def output_size(self, width: int, height: int):
        """(width, height) of the resized image (torchvision's _compute_resized_output_size)."""
        if len(self.size) == 2:
            return self.size[1], self.size[0]
        short, long = (width, height) if width <= height else (height, width)
        new_short, new_long = self.size[0], int(self.size[0] * long / short)
        return (new_short, new_long) if width <= height else (new_long, new_short)

    def __call__(self, img):
        from PIL import Image
        size = self.output_size(*img.size)
        if size == img.size:
            return img
        return img.resize(size, Image.BILINEAR)


class CenterCrop:
    """torchvision.transforms.CenterCrop on a PIL image: size is an int or (height, width); the box starts at
    int(round((side - crop) / 2)), and a crop larger than the image is padded with zeros around it, as torchvision pads."""

    def __init__(self, size: Union[int, Sequence[int]]):
        if isinstance(size, int):
            size = [size]
        if len(size) not in (1, 2):
            raise ValueError(f"CenterCrop size must be an int or a list of 1 or 2 ints, got {size!r}")
        self.height, self.width = (int(size[0]), int(size[-1]))

    @staticmethod
    def _start(side: int, crop: int) -> int:
        if crop > side:                  # torchvision pads (crop - side) // 2 before the image and crops from 0
            return -((crop - side) // 2)
        return int(round((side - crop) / 2.0))

    def __call__(self, img):
        w, h = img.size
        left, top = self._start(w, self.width), self._start(h, self.height)
        return img.crop((left, top, left + self.width, top + self.height))


TRANSFORMS = {"Resize": Resize, "CenterCrop": CenterCrop}


def build_transforms(transform_opts: Sequence[Mapping]) -> List:
    """The PIL transforms of a `video_transform` list, in order.  ToTensor and Normalize are accepted and left out; any
    other type raises NotImplementedError."""
    out = []
    for opt in transform_opts:
        opt = dict(opt)
        kind = opt.pop("type")
        if kind in _TENSOR_TRANSFORMS:
            continue
        if kind not in TRANSFORMS:
            raise NotImplementedError(f"video_transform type {kind!r} is not supported (Resize, CenterCrop, ToTensor and "
                                      "Normalize are)")
        out.append(TRANSFORMS[kind](**opt))
    return out


class SingleVideoPointDataset:
    """frame_point_dataset.py's dataset at test time.  opt: the config's `datasets` entry (path, prompt, num_frames,
    total_frames, video_transform, tap_path).

      * `select_id`: formats.select_frame_idx(0, min(#frames, total_frames), num_frames) over the sorted frame directory;
      * `get_frames()`: the selected frames as RGB PIL images after the Resize / CenterCrop transforms;
      * `get_conditions(tap_path=None)`: the TAP file's tracks at select_id, with img_size = (width, height) of the
        transformed frames; without a path, the conditions of the config's own `tap_path` (None when it has none)."""

    def __init__(self, opt: Mapping):
        self.opt = opt
        self.total_frames = sorted(Path(opt["path"]).iterdir())
        self.select_id = formats.select_frame_idx(0, min(len(self.total_frames), opt["total_frames"]), opt["num_frames"])
        self.video = [self.total_frames[i] for i in self.select_id]
        self.prompt = opt["prompt"]
        self.num_video = opt.get("dataset_enlarge_ratio", 1)
        self.video_transform = build_transforms(opt["video_transform"])
        self._frames = [self._load(path) for path in self.video]
        sizes = sorted({f.size for f in self._frames})
        if len(sizes) != 1:
            raise ValueError(f"the selected frames differ in size after the transforms: {sizes}")
        self.size_x, self.size_y = sizes[0]
        tap_path = opt.get("tap_path")
        self.condition = self.get_conditions(tap_path) if tap_path is not None else None

    def _load(self, path):
        from PIL import Image
        with Image.open(path) as im:
            frame = im.convert("RGB")
        for t in self.video_transform:
            frame = t(frame)
        return frame

    def __len__(self):
        return self.num_video

    def get_frames(self) -> List:
        """The selected frames (fresh copies: callers may draw on them)."""
        return [f.copy() for f in self._frames]

    def get_conditions(self, tap_path: Optional[str] = None) -> Optional[Dict]:
        if tap_path is None:
            return self.condition
        return formats.load_tap(tap_path, select_id=self.select_id, img_size=(self.size_x, self.size_y))
