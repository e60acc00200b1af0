"""Host side of the region prompts (visual-prompt task, SURVEY.md section 8 f3).

`region_pooling` of the reference (visual_prompt_module/context_cluster.py:333-400) does two things: it DRAWS 256 sample
points per region mask on the host (`rand_sample_repeat`, context_cluster.py:31-40: torch.randint / torch.randperm on the
global CPU generator) and it samples + averages the projector's feature map at those points.  The second part is the
CUDA kernel `psalm_region_pool`; the first part is restated here with the same calls in the same order, so that a
caller who seeds the generator like the reference gets the reference's points."""
import torch

NUM_SAMPLE_POINT = 256   # llava_phi.py:162


def sample_region_points(region_masks, num_sample_point=NUM_SAMPLE_POINT):
    """region_masks [K,H,W] (bool / 0-1, host or device) -> [K, num_sample_point, 2] fp32 host tensor of normalised
    (y / H, x / W) positions of mask pixels: all of them plus random repeats when the mask is small, a random subset
    when it is large (context_cluster.py:31-40, :349-352)."""
    region_masks = region_masks.cpu()
    if region_masks.shape[0] == 0:
        return torch.zeros(0, num_sample_point, 2)
    wh = torch.tensor([region_masks[0].shape[0], region_masks[0].shape[1]])[None]
    out = []
    for m in region_masks:
        x = m.nonzero() / wh
        if x.shape[0] == 0:
            raise ValueError("empty region mask (the reference prints 'error' and then fails in torch.randint)")
        if x.shape[0] < num_sample_point:
            idx = torch.randint(0, x.shape[0], (num_sample_point - x.shape[0],))
            x = torch.cat((x, x[idx]), dim=0)
        elif x.shape[0] > num_sample_point:
            x = x[torch.randperm(x.shape[0])[:num_sample_point], :]
        out.append(x)
    return torch.stack(out).float()


def draw_point_indices(counts, num_sample_point=NUM_SAMPLE_POINT):
    """The random part of `sample_region_points` for masks with `counts` set pixels: [K, num_sample_point] int32 indices
    into each mask's `nonzero()` rows, drawn with the same calls in the same order on the global CPU generator, so that
    `m.nonzero()[idx] / wh` equals `sample_region_points` from the same generator state.  The masks themselves stay on the
    device (kernels.region_points_gather turns the indices into points)."""
    out = []
    for n in counts:
        n = int(n)
        if n == 0:
            raise ValueError("empty region mask (the reference prints 'error' and then fails in torch.randint)")
        if n < num_sample_point:
            idx = torch.cat((torch.arange(n), torch.randint(0, n, (num_sample_point - n,))))
        elif n > num_sample_point:
            idx = torch.randperm(n)[:num_sample_point]
        else:
            idx = torch.arange(n)
        out.append(idx)
    return torch.stack(out).to(torch.int32)


# ---- visual prompts: clicks, scribbles, boxes and masks at the original image size (COCO-Interactive) ------------------
# enhance_with_circles radius per kind (coco_instance_mapper.py:247-249); boxes and masks are resized as they are
VISUAL_PROMPT_RADIUS = {"point": 10, "scribble": 5, "box": 0, "mask": 0}


def _rle_has_foreground(counts):
    """Whether a COCO compressed RLE string (rleFrString's LEB128-like code) has a non-zero run of ones."""
    s = counts.encode("ascii") if isinstance(counts, str) else bytes(counts)
    runs, p = [], 0
    while p < len(s):
        x, k, more = 0, 0, True
        while more:
            c = s[p] - 48
            x |= (c & 0x1f) << (5 * k)
            more = bool(c & 0x20)
            p += 1
            k += 1
            if not more and c & 0x10:
                x |= -1 << (5 * k)
        if len(runs) > 2:
            x += runs[-2]
        runs.append(x)
    return any(n > 0 for n in runs[1::2])


def _source_masks(prompts, height, width, device):
    """(uint8 [K,height,width] prompt masks on `device`, int32 [K] radii) of K (kind, source) pairs; ValueError for an
    unknown kind, a source of the wrong form or size, or an empty source, before anything is launched."""
    from . import rle
    K = len(prompts)
    if K == 0:
        raise ValueError("visual_prompts: no regions")
    src = torch.zeros((K, height, width), dtype=torch.uint8, device=device)
    radius, rles = [], []
    for k, p in enumerate(prompts):
        if not isinstance(p, (tuple, list)) or len(p) != 2:
            raise ValueError("visual prompt %d: expected a (kind, source) pair" % k)
        kind, s = p
        if kind not in VISUAL_PROMPT_RADIUS:
            raise ValueError("visual prompt %d: kind %r is not one of %s" % (k, kind, sorted(VISUAL_PROMPT_RADIUS)))
        r = VISUAL_PROMPT_RADIUS[kind]
        radius.append(r)
        if isinstance(s, dict):                    # COCO RLE at the original size
            if [int(v) for v in s.get("size", ())] != [height, width]:
                raise ValueError("visual prompt %d: RLE size %s, the image is %dx%d" % (k, s.get("size"), height, width))
            if not isinstance(s.get("counts"), (str, bytes, bytearray)) or not _rle_has_foreground(s["counts"]):
                raise ValueError("visual prompt %d: empty source mask" % k)
            rles.append((k, s))
        elif isinstance(s, torch.Tensor):          # binary [H0, W0], host or device
            if tuple(s.shape) != (height, width):
                raise ValueError("visual prompt %d: mask %s, the image is %dx%d" % (k, tuple(s.shape), height, width))
            s = s.to(device).to(torch.uint8)       # binary_mask.astype(np.uint8) (:27)
            if not bool((s == 1).any() if r > 0 else (s != 0).any()):   # only pixels equal to 1 seed a disk (:30)
                raise ValueError("visual prompt %d: empty source mask" % k)
            src[k] = s
        elif kind == "point" and len(s) == 2:      # a click (row, col)
            y, x = (int(v) for v in s)
            if not (0 <= y < height and 0 <= x < width):
                raise ValueError("visual prompt %d: point %s outside the %dx%d image" % (k, (y, x), height, width))
            src[k, y, x] = 1
        elif kind == "box" and len(s) == 4:        # (min_row, min_col, max_row, max_col), half-open (bulid_COCO_...:72)
            y0, x0, y1, x1 = (int(v) for v in s)
            y0, x0, y1, x1 = max(0, y0), max(0, x0), min(height, y1), min(width, x1)
            if y1 <= y0 or x1 <= x0:
                raise ValueError("visual prompt %d: empty source mask (box %s)" % (k, tuple(s)))
            src[k, y0:y1, x0:x1] = 1
        else:
            raise ValueError("visual prompt %d: a %s takes an RLE dict, a [H, W] tensor%s" % (
                k, kind, {"point": " or a (row, col) pixel", "box": " or (min_row, min_col, max_row, max_col)"}.get(kind, "")))
    if rles:
        dec = rle.decode([s for _, s in rles], device)
        for i, (k, _) in enumerate(rles):
            src[k] = dec[i]
    return src, torch.tensor(radius, dtype=torch.int32).to(device)


def rasterize_visual_prompts(prompts, height, width, resized_hw, padded_hw, device):
    """K visual prompts (kind, source) of an image of original size (height, width) -> the region masks the reference
    mapper gives (coco_instance_mapper.py:233-251: decode, enhance_with_circles for points and scribbles, NEAREST resize
    to `resized_hw`, zero padding to `padded_hw`) as (bits, row_prefix, count) in the layout `region_points_gather`
    reads, on `device`.  `kind` is "point", "scribble", "box" or "mask"; `source` is a COCO RLE dict at the original
    size, a binary [height, width] tensor, a (row, col) pixel for a point or a (min_row, min_col, max_row, max_col) box."""
    from . import kernels
    from .image_processor import nearest_pad_tables
    src, radius = _source_masks(prompts, int(height), int(width), device)
    rows, cols = nearest_pad_tables(int(height), int(width), resized_hw, padded_hw)
    return kernels.visual_prompt_raster(src, radius, rows.to(device), cols.to(device))


def region_inputs(seg_info, region_points=None, attr="region_masks"):
    """seg_info: list of dicts with 'instances' (`.region_masks.tensor` [K,H,W], llava_phi.py:792; the DAVIS variant reads
    `.vp_region_masks`, :1664) -> (points [R,P,2] fp32, region_image [R] int32, counts).  `region_points`: optional
    per-sample list of pre-drawn points."""
    pts, img, counts = [], [], []
    for b, info in enumerate(seg_info):
        p = region_points[b] if region_points is not None else sample_region_points(getattr(info["instances"], attr).tensor)
        pts.append(p.float().cpu())
        img += [b] * p.shape[0]
        counts.append(int(p.shape[0]))
    return torch.cat(pts, 0).contiguous(), torch.tensor(img, dtype=torch.int32), tuple(counts)
