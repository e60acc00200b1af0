"""COCO run-length encoding of instance masks on the device (SURVEY.md section 8 f1).

The output is byte-identical to pycocotools (`pycocotools.mask.encode` on the Fortran-ordered [H, W, n] uint8 stack),
which is not a dependency of this package.  Dense fp32 instance masks of a 1024^2 image with 100 instances are 419 MB;
their RLE strings are a few kB per mask, and they are the form COCO evaluators consume.

Two forms:
  * pycocotools dicts {"size": [H, W], "counts": bytes} (`encode`, `decode`, `instances_to_coco_json`);
  * the device form (`encode_device`): dict(size=(H, W), chars uint8 [bytes] (the strings back to back),
    offsets int64 [n+1], area int64 [n], bbox float64 [n, 4]), all CUDA tensors - what `dist.gather_rle` moves
    between ranks and what a GPU-side consumer reads.
No CPU path: masks must be CUDA tensors.
"""
import torch

from . import _lib
from . import kernels


def _stack_shape(masks):
    if masks.dim() == 2:
        return masks.unsqueeze(0)
    if masks.dim() != 3:
        raise _lib.PsalmKernelError("rle: masks are [n, H, W] or [H, W], got %s" % (tuple(masks.shape),))
    return masks


def encode_device(masks):
    """[n,H,W] / [H,W] CUDA masks (float32, uint8 or bool; non-zero = foreground), or a list of [k,H,W] tensors of one
    size, -> the device form.  Empty input launches nothing."""
    parts = [_stack_shape(masks)] if isinstance(masks, torch.Tensor) else [_stack_shape(m) for m in masks]
    if not parts:
        raise _lib.PsalmKernelError("rle.encode_device: no masks (pass an [0, H, W] tensor for an empty batch)")
    _lib.require_cuda(*parts)
    H, W = (int(s) for s in parts[0].shape[1:])
    parts = [p.contiguous() for p in parts if p.shape[0] > 0]
    dev = parts[0].device if parts else None
    if not parts:
        dev = (masks if isinstance(masks, torch.Tensor) else masks[0]).device
        return dict(size=(H, W), chars=torch.empty(0, dtype=torch.uint8, device=dev),
                    offsets=torch.zeros(1, dtype=torch.int64, device=dev),
                    area=torch.empty(0, dtype=torch.int64, device=dev),
                    bbox=torch.empty((0, 4), dtype=torch.float64, device=dev))
    out = kernels.rle_encode(parts[0] if len(parts) == 1 else parts)
    out["size"] = (H, W)
    return out


def to_dicts(dev_form):
    """Device form -> list of pycocotools dicts (one device-to-host copy of the strings and offsets)."""
    H, W = dev_form["size"]
    chars = dev_form["chars"].cpu().numpy().tobytes()
    offs = dev_form["offsets"].cpu().tolist()
    return [{"size": [H, W], "counts": chars[offs[i]:offs[i + 1]]} for i in range(len(offs) - 1)]


def encode(masks):
    """pycocotools.mask.encode(np.asfortranarray(masks.permute(1, 2, 0).cpu().numpy().astype(np.uint8))) for a
    [n,H,W] CUDA tensor (a list of dicts; a [H,W] mask gives a list of one)."""
    return to_dicts(encode_device(masks))


def _from_dicts(rles, device):
    if not rles:
        raise _lib.PsalmKernelError("rle: empty list of RLE dicts")
    H, W = (int(s) for s in rles[0]["size"])
    strs = []
    for r in rles:
        if tuple(int(s) for s in r["size"]) != (H, W):
            raise _lib.PsalmKernelError("rle: every RLE of one call needs the same size")
        c = r["counts"]
        if isinstance(c, str):
            c = c.encode("ascii")
        if not isinstance(c, (bytes, bytearray)):
            raise _lib.PsalmKernelError("rle: counts must be a compressed string (bytes or str)")
        strs.append(bytes(c))
    offs = [0]
    for s in strs:
        offs.append(offs[-1] + len(s))
    blob = b"".join(strs)
    chars = torch.frombuffer(bytearray(blob), dtype=torch.uint8).to(device) if blob else \
        torch.empty(0, dtype=torch.uint8, device=device)
    return (H, W), chars, torch.tensor(offs, dtype=torch.int64).to(device)


def decode(rles, device="cuda"):
    """pycocotools dicts (bytes or str counts, one size) or the device form -> uint8 [n,H,W] on the device."""
    if isinstance(rles, dict):
        (H, W), chars, offsets = rles["size"], rles["chars"], rles["offsets"]
    else:
        if len(rles) == 0:
            return torch.empty((0, 0, 0), dtype=torch.uint8, device=device)
        (H, W), chars, offsets = _from_dicts(rles, device)
    if offsets.numel() == 1:
        return torch.empty((0, H, W), dtype=torch.uint8, device=offsets.device)
    return kernels.rle_decode(chars, offsets, H, W)


def _device_form(rles, device):
    if isinstance(rles, dict):
        return rles
    if len(rles) == 0:
        return None
    return encode_device(decode(rles, device))


def area(rles, device="cuda"):
    """rleArea: foreground pixels per mask, int64 [n] on the device."""
    d = _device_form(rles, device)
    return d["area"] if d is not None else torch.empty(0, dtype=torch.int64, device=device)


def to_bbox(rles, device="cuda"):
    """rleToBbox: [x, y, w, h] float64 [n, 4] on the device, the tight box of the foreground (zeros when empty)."""
    d = _device_form(rles, device)
    return d["bbox"] if d is not None else torch.empty((0, 4), dtype=torch.float64, device=device)


def instances_to_coco_json(instances, img_id, rles=None):
    """detectron2's `instances_to_coco_json` with the masks encoded on the device: one record per instance with
    image_id, category_id, bbox (from `pred_boxes`, XYXY -> XYWH, as detectron2 does; not the mask box), score and
    segmentation ({"size", "counts"} with str counts).  `rles`: the instances' masks already encoded (e.g.
    `instances.pred_masks_rle` of an `eval_seg(..., mask_format="rle")` result); encoded here otherwise."""
    n = len(instances)
    if n == 0:
        return []
    boxes = instances.pred_boxes.tensor.detach().cpu().float().clone()
    boxes[:, 2:] -= boxes[:, :2]
    boxes = boxes.tolist()
    scores = instances.scores.tolist()
    classes = instances.pred_classes.tolist()
    if rles is None:
        rles = instances.pred_masks_rle if instances.has("pred_masks_rle") else encode(instances.pred_masks)
    results = []
    for k in range(n):
        seg = {"size": list(rles[k]["size"]), "counts": rles[k]["counts"].decode("utf-8")}
        results.append({"image_id": img_id, "category_id": classes[k], "bbox": boxes[k], "score": scores[k],
                        "segmentation": seg})
    return results
