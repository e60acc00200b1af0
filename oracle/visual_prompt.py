"""TEST INFRASTRUCTURE — plain numpy / Pillow restatement of the reference mapper's region-mask path for visual prompts
(psalm/model/datasets_mapper/coco_instance_mapper.py:17-33, :233-251), used by the tests and tools/bench_interactive.py:

    region_mask = decode(anno[used_mask_type])                        # 0/1 uint8 at the original size
    if point or scribble: region_mask = enhance_with_circles(region_mask, 10 or 5)
    scale_region_mask = transforms.apply_segmentation(region_mask)    # Pillow NEAREST resize, FixedSizeCrop zero pad

`enhance_with_circles` is the reference's algorithm (one full-image float64 distance test per seed pixel): it is what a
host-side mapper pays per region.  `dilate` is the same set computed with a disk structuring element, for the large
tests; tests/test_interactive_cpu.py pins both to tests/golden/visual_prompts.npz, made by the unmodified reference."""
import numpy as np

from oracle.davis_loop import apply_segmentation

RADIUS = {"point": 10, "scribble": 5, "box": 0, "mask": 0}   # coco_instance_mapper.py:247-249


def draw_circle(mask, center, radius):
    """coco_instance_mapper.py:17-20."""
    y, x = np.ogrid[:mask.shape[0], :mask.shape[1]]
    distance = np.sqrt((x - center[1]) ** 2 + (y - center[0]) ** 2)
    mask[distance <= radius] = 1


def enhance_with_circles(binary_mask, radius=5):
    """coco_instance_mapper.py:23-33."""
    binary_mask = np.asarray(binary_mask).astype(np.uint8)
    output_mask = np.zeros_like(binary_mask, dtype=np.uint8)
    for point in np.argwhere(binary_mask == 1):
        draw_circle(output_mask, (point[0], point[1]), radius)
    return output_mask


def disk(radius):
    """bool [2r+1, 2r+1]: dx^2 + dy^2 <= r^2."""
    d = np.arange(-radius, radius + 1)
    return d[:, None] ** 2 + d[None, :] ** 2 <= radius * radius


def dilate(binary_mask, radius):
    """enhance_with_circles(binary_mask, radius) as a binary dilation by `disk(radius)` (zeros outside the image)."""
    from scipy.ndimage import binary_dilation
    seeds = np.asarray(binary_mask).astype(np.uint8) == 1
    return binary_dilation(seeds, structure=disk(radius)).astype(np.uint8) if seeds.any() else seeds.astype(np.uint8)


def paint_box(height, width, box):
    """datasets/bulid_COCO_Interactivate.py:72: mask[min_row:max_row, min_col:max_col] = 1."""
    m = np.zeros((height, width), np.uint8)
    y0, x0, y1, x1 = box
    m[max(0, y0):min(height, y1), max(0, x0):min(width, x1)] = 1
    return m


def region_mask(kind, mask, resized_hw, padded_hw, literal=False):
    """The region mask the mapper gives for a prompt mask `mask` (0/1 uint8 at the original size) of `kind`: bool
    [Hp, Wp].  `literal` runs the reference's per-seed disks instead of the dilation."""
    r = RADIUS[kind]
    if r:
        mask = enhance_with_circles(mask, r) if literal else dilate(mask, r)
    return apply_segmentation(np.asarray(mask, np.uint8), resized_hw, padded_hw) != 0
