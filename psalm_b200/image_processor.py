"""Image processors = the `vision_tower.image_processor` dict of the reference (language_model/llava_phi.py:66-69,
keys panoptic | instance | semantic), consumed by the eval datasets as `processor.preprocess(data_dict, ...)`
(psalm/train/train_datasets.py:203-207).

Restates the INFERENCE part of the reference mappers (datasets_mapper/coco_panoptic_mapper.py:134-164 and siblings;
build_transform_gen :81-89): read the image, ResizeShortestEdge(short = max = IMAGE_SIZE), FixedSizeCrop(IMAGE_SIZE^2,
pad value 128, padding mask from a ones-mask padded with 0), CHW tensor, `(image - pixel_mean) / pixel_std`.
detectron2's transforms (un-vendored third party, version unpinned upstream) are restated from their documented
semantics: new size = round-half-up of the scaled size, PIL bilinear resampling for uint8 images, padding at the
bottom / right.  Ground-truth handling (panoptic PNGs, polygons) belongs to training / evaluation and is not restated.

On top of the reference contract, `preprocess` also returns `image_u8` (the padded uint8 CHW image): `PSALM.eval_seg`
accepts it directly and normalises on the device (csrc/preproc.cu), a 4x smaller upload.  `preprocess_device` moves the
resize and the padding to the device too, with Pillow's 8-bit resampling arithmetic restated exactly (`pil_bilinear_resize`:
bit-identical to `Image.resize(BILINEAR)`, tests/test_surface_cpu.py)."""
import numpy as np
import torch

PIXEL_MEAN = (123.675, 116.28, 103.53)   # coco_panoptic_mapper.py:118-119
PIXEL_STD = (58.395, 57.12, 57.375)


def resize_shortest_edge_shape(h, w, short, max_size):
    """detectron2 ResizeShortestEdge.get_output_shape: scale the short side to `short`, cap the long side at
    `max_size`, round half up."""
    scale = short * 1.0 / min(h, w)
    if h < w:
        newh, neww = short, scale * w
    else:
        newh, neww = scale * h, short
    if max(newh, neww) > max_size:
        scale = max_size * 1.0 / max(newh, neww)
        newh, neww = newh * scale, neww * scale
    return int(newh + 0.5), int(neww + 0.5)


_PRECISION_BITS = 32 - 8 - 2      # Pillow: src/libImaging/Resample.c, 8 bits per channel
_COEFFS = {}


def _pil_bilinear_coeffs(in_size, out_size, device):
    """Dense [out_size, in_size] matrix of the INTEGER coefficients Pillow's 8-bit resampler uses for the BILINEAR filter
    over the whole image (Resample.c: precompute_coeffs + normalize_coeffs_8bpc): triangle filter of support
    max(scale, 1) around the source centre (xx + 0.5) * scale, normalised in double, scaled by 2^22 and rounded half away
    from zero.  Cached per (sizes, device)."""
    key = (in_size, out_size, str(device))
    if key not in _COEFFS:
        scale = in_size / out_size
        filterscale = max(scale, 1.0)
        support = 1.0 * filterscale
        K = np.zeros((out_size, in_size), dtype=np.float64)
        for xx in range(out_size):
            center = (xx + 0.5) * scale
            xmin = max(int(center - support + 0.5), 0)
            xmax = min(int(center + support + 0.5), in_size)
            arg = (np.arange(xmax - xmin) + xmin - center + 0.5) / filterscale
            w = np.where(np.abs(arg) < 1.0, 1.0 - np.abs(arg), 0.0)
            ww = w.sum()
            K[xx, xmin:xmax] = w / ww if ww != 0.0 else w
        K = np.trunc(0.5 + K * (1 << _PRECISION_BITS))      # all bilinear coefficients are >= 0
        _COEFFS[key] = torch.from_numpy(K).to(device)
    return _COEFFS[key]


def pil_bilinear_resize(image_hwc_u8, out_h, out_w):
    """uint8 [H,W,C] tensor (any device) -> uint8 [out_h,out_w,C] with the bits of
    `PIL.Image.resize((out_w, out_h), Image.BILINEAR)`: Pillow's two passes (horizontal, then vertical, uint8 in between),
    each `clip8((sum_x pixel * coeff + 2^21) >> 22)`.  The sums are integers below 2^34, so float64 GEMMs evaluate them
    exactly in any summation order - on the GPU this is two small DGEMMs instead of a host-side resize of every image."""
    x = image_hwc_u8.double()
    H, W, _ = x.shape
    half, one = float(1 << (_PRECISION_BITS - 1)), float(1 << _PRECISION_BITS)
    if W != out_w:
        x = torch.einsum("hwc,ow->hoc", x, _pil_bilinear_coeffs(W, out_w, x.device))
        x = torch.floor((x + half) / one).clamp_(0, 255)
    if H != out_h:
        x = torch.einsum("hwc,oh->owc", x, _pil_bilinear_coeffs(H, out_h, x.device))
        x = torch.floor((x + half) / one).clamp_(0, 255)
    return x.to(torch.uint8)


def pil_nearest_index(in_size, out_size):
    """int64 [out_size]: the source index of every output column (or row) of `PIL.Image.resize(..., Image.NEAREST)`, -1
    where Pillow leaves the pixel unset (0).  Pillow's ImagingScaleAffine (Geometry.c) starts at scale / 2 and ADDS the
    scale (in double) once per output pixel, truncating each sum; evaluating (x + 0.5) * scale directly instead differs
    from Pillow at some sizes (tests/test_video_cpu.py compares both axes with Pillow)."""
    scale = in_size / out_size
    idx = np.empty(out_size, dtype=np.int64)
    xo = scale * 0.5
    for x in range(out_size):
        xin = -1 if xo < 0.0 else int(xo)
        idx[x] = xin if xin < in_size else -1
        xo += scale
    return idx


def nearest_pad_tables(height, width, resized_hw, padded_hw):
    """detectron2 `ResizeTransform.apply_segmentation` (Pillow NEAREST from (height, width) to `resized_hw`) followed by
    FixedSizeCrop's zero padding to `padded_hw` (seg_pad_value=0, coco_*_mapper.py build_transform_gen), as source-row
    and source-column tables: int32 [Hp] and [Wp], -1 = zero."""
    (oh, ow), (Hp, Wp) = resized_hw, padded_hw
    rows = np.full(Hp, -1, dtype=np.int32)
    cols = np.full(Wp, -1, dtype=np.int32)
    rows[:oh] = pil_nearest_index(height, oh)
    cols[:ow] = pil_nearest_index(width, ow)
    return torch.from_numpy(rows), torch.from_numpy(cols)


class SegImageProcessor:
    """One class for the three mappers: they differ in ground-truth handling only (not restated)."""

    def __init__(self, image_size=1024, task="panoptic", pad_value=128.0):
        self.image_size, self.task, self.pad_value = int(image_size), task, float(pad_value)
        self.pixel_mean = torch.tensor(PIXEL_MEAN).view(-1, 1, 1)
        self.pixel_std = torch.tensor(PIXEL_STD).view(-1, 1, 1)

    def _read(self, dataset_dict):
        if "image_array" in dataset_dict:           # HWC uint8 RGB, already decoded
            return np.asarray(dataset_dict["image_array"], dtype=np.uint8)
        from PIL import Image
        with Image.open(dataset_dict["file_name"]) as im:
            return np.asarray(im.convert("RGB"), dtype=np.uint8)

    def preprocess(self, dataset_dict, region_mask_type=None, mask_format="polygon"):
        d = dict(dataset_dict)
        image = self._read(d)
        h, w = image.shape[:2]
        d.setdefault("height", h)
        d.setdefault("width", w)
        S = self.image_size
        nh, nw = resize_shortest_edge_shape(h, w, S, S)
        if (nh, nw) != (h, w):
            from PIL import Image
            image = np.asarray(Image.fromarray(image).resize((nw, nh), Image.BILINEAR))
        padded = np.full((S, S, 3), self.pad_value, dtype=np.float32).astype(np.uint8)
        padded[:nh, :nw] = image[:S, :S]
        padding_mask = np.ones((S, S), dtype=bool)
        padding_mask[:nh, :nw] = False               # ~ (ones-mask padded with 0)
        u8 = torch.as_tensor(np.ascontiguousarray(padded.transpose(2, 0, 1)))
        d["image_u8"] = u8
        d["image"] = (u8 - self.pixel_mean) / self.pixel_std
        d["padding_mask"] = torch.as_tensor(padding_mask)
        d["transforms"] = None
        return d


    def preprocess_device(self, dataset_dict, device="cuda"):
        """`preprocess` with the resize, the padding and (inside `PSALM.eval_seg`, csrc/preproc.cu) the normalisation on
        the DEVICE: the decoded image is uploaded as it is (H x W x 3 bytes, usually far fewer than the padded
        1024^2 x 3), resized with Pillow's exact 8-bit arithmetic (`pil_bilinear_resize`), padded with 128 at the bottom /
        right.  Returns the same dict as `preprocess` without the float `image`; `image_u8` [3,S,S] lives on `device`
        and is bit-identical to the host path's."""
        d = dict(dataset_dict)
        image = self._read(d)
        h, w = image.shape[:2]
        d.setdefault("height", h)
        d.setdefault("width", w)
        S = self.image_size
        nh, nw = resize_shortest_edge_shape(h, w, S, S)
        x = torch.as_tensor(np.ascontiguousarray(image)).to(device, non_blocking=True)
        if (nh, nw) != (h, w):
            x = pil_bilinear_resize(x, nh, nw)
        padded = torch.full((3, S, S), int(self.pad_value), dtype=torch.uint8, device=device)
        padded[:, :nh, :nw] = x[:S, :S].permute(2, 0, 1)
        padding_mask = torch.ones((S, S), dtype=torch.bool)
        padding_mask[:nh, :nw] = False
        d["image_u8"] = padded
        d["padding_mask"] = padding_mask
        d["transforms"] = None
        return d


def build_image_processors(image_size=1024):
    """The dict `PSALMModel.__init__` attaches to the vision tower (llava_phi.py:66-69)."""
    return {k: SegImageProcessor(image_size, k) for k in ("panoptic", "instance", "semantic")}
