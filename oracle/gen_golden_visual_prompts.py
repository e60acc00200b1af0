"""TEST INFRASTRUCTURE — generates tests/golden/visual_prompts.npz by running the UNMODIFIED reference's
`enhance_with_circles` (psalm/model/datasets_mapper/coco_instance_mapper.py:17-33, imported through oracle/ref_shims.py:
cv2 is real, detectron2 and pycocotools are shimmed) on seeded prompt masks of all four kinds at COCO-like sizes:
clicks and scribbles touching the borders and corners, boxes (bulid_COCO_Interactivate.py:72) and masks, radius 10
(point) and 5 (scribble).  Boxes and masks are not dilated by the mapper; their output is the input.

    PSALM_REFERENCE_ROOT=<reference checkout> python oracle/gen_golden_visual_prompts.py

Stored per case i: kind_i, src_i / out_i (np.packbits along the rows of the [H, W] 0/1 masks) and shape_i."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_shims  # noqa: E402
from oracle.visual_prompt import RADIUS, paint_box  # noqa: E402

SIZES = [(480, 640), (640, 427), (333, 500), (1333, 1000)]


def scribble(rng, H, W, n, through=None):
    """A random walk of n steps (8-neighbourhood), clipped to the image, started at `through` or a random pixel."""
    y, x = through if through is not None else (int(rng.integers(H)), int(rng.integers(W)))
    m = np.zeros((H, W), np.uint8)
    for _ in range(n):
        m[y, x] = 1
        y = int(np.clip(y + rng.integers(-1, 2), 0, H - 1))
        x = int(np.clip(x + rng.integers(-1, 2), 0, W - 1))
    return m


def blob(rng, H, W):
    yy, xx = np.ogrid[:H, :W]
    cy, cx = rng.integers(H), rng.integers(W)
    ry, rx = rng.integers(5, H // 4), rng.integers(5, W // 4)
    return (((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 <= 1).astype(np.uint8)


def cases(rng, H, W):
    out = []
    for corner in ((0, 0), (H - 1, W - 1), (0, W - 1), (H - 1, 0)):   # single clicks in the corners
        m = np.zeros((H, W), np.uint8)
        m[corner] = 1
        out.append(("point", m))
    m = np.zeros((H, W), np.uint8)                                   # three clicks, one on an edge
    m[rng.integers(H), 3] = m[rng.integers(H), rng.integers(W)] = m[H - 2, rng.integers(W)] = 1
    out.append(("point", m))
    out.append(("scribble", scribble(rng, H, W, 300, (0, int(rng.integers(W))))))        # from the top edge
    out.append(("scribble", scribble(rng, H, W, 120, (H - 1, W - 1))))                   # from a corner
    out.append(("scribble", scribble(rng, H, W, 200)))
    y0, x0 = int(rng.integers(H // 2)), int(rng.integers(W // 2))
    out.append(("box", paint_box(H, W, (y0, x0, y0 + int(rng.integers(1, H // 2)), x0 + int(rng.integers(1, W // 2))))))
    out.append(("box", paint_box(H, W, (H - 40, W - 60, H + 10, W + 10))))             # clipped at the border
    out.append(("mask", blob(rng, H, W)))
    m = blob(rng, H, W)
    m[0, :] = 1                                                                         # touches the first row
    out.append(("mask", m))
    return out


def main():
    ref_shims.install()
    from psalm.model.datasets_mapper.coco_instance_mapper import enhance_with_circles
    rng = np.random.default_rng(2024)
    gold = {}
    i = 0
    for H, W in SIZES:
        for kind, src in cases(rng, H, W):
            out = enhance_with_circles(src, RADIUS[kind]) if RADIUS[kind] else src
            gold["kind_%d" % i] = np.array(kind)
            gold["shape_%d" % i] = np.array([H, W], np.int64)
            gold["src_%d" % i] = np.packbits(src.astype(bool), axis=1)
            gold["out_%d" % i] = np.packbits(np.asarray(out).astype(bool), axis=1)
            i += 1
            print(H, W, kind, int(src.sum()), int(np.asarray(out).sum()))
    gold["n"] = np.array(i)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "visual_prompts.npz"), **gold)


if __name__ == "__main__":
    main()
