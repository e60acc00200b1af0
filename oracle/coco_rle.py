"""COCO run-length encoding in plain numpy: a restatement of pycocotools' maskApi.c (rleEncode, rleToString,
rleFrString, rleDecode, rleArea, rleToBbox) that the tests compare the device encoder (csrc/rle.cu) against.

pycocotools is third-party and not a dependency of this project; this module restates its contract, it does not call
it (the tests cross-check the two when pycocotools happens to be importable).  The contract, per mask [H, W]:
  * pixels are taken in column-major order j = x*H + y; a pixel is foreground iff it is non-zero;
  * counts are the lengths of alternating runs, background first (the first count may be 0), uint32;
  * the string form encodes value v_i = cnt[i] - cnt[i-2] for i > 2, else cnt[i], as 5-bit groups, low bits first,
    continuing while (group & 0x10) ? v != -1 : v != 0 after an arithmetic shift, with bit 0x20 set on continued
    groups and 48 added to every group;
  * area is the sum of the odd runs; bbox [x, y, w, h] is the tight box of the foreground, zeros when empty.
"""
import numpy as np


def encode(mask):
    """rleEncode: [H, W] mask -> counts (list of int)."""
    f = (np.asarray(mask) != 0).ravel(order="F").astype(np.int8)
    trans = np.flatnonzero(np.diff(np.concatenate(([0], f))) != 0)
    bounds = np.concatenate(([0], trans, [f.size]))
    return [int(c) for c in np.diff(bounds)]


def to_string(counts):
    """rleToString: counts -> bytes."""
    out = bytearray()
    for i, c in enumerate(counts):
        x = int(c) - (int(counts[i - 2]) if i > 2 else 0)
        more = True
        while more:
            g = x & 0x1F
            x >>= 5   # Python's >> on int is an arithmetic shift
            more = x != -1 if g & 0x10 else x != 0
            if more:
                g |= 0x20
            out.append(g + 48)
    return bytes(out)


def fr_string(s):
    """rleFrString: bytes (or str) -> counts."""
    if isinstance(s, str):
        s = s.encode("ascii")
    counts, p = [], 0
    while p < len(s) and s[p]:
        x, k, more = 0, 0, True
        while more:
            c = s[p] - 48
            x |= (c & 0x1F) << (5 * k)
            more = bool(c & 0x20)
            p += 1
            k += 1
            if not more and c & 0x10:
                x |= -1 << (5 * k)
        if len(counts) > 2:
            x += counts[-2]
        counts.append(x & 0xFFFFFFFF)
    return counts


def decode(counts, H, W):
    """rleDecode: counts -> [H, W] uint8."""
    vals = np.arange(len(counts)) % 2
    f = np.repeat(vals.astype(np.uint8), np.asarray(counts, dtype=np.int64))
    return f.reshape((W, H)).T.copy()


def area(counts):
    """rleArea: sum of the odd runs."""
    return int(sum(counts[1::2]))


def to_bbox(counts, H, W):
    """rleToBbox: [x, y, w, h] as floats; zeros for an empty mask."""
    m = len(counts) // 2 * 2
    if m == 0:
        return [0.0, 0.0, 0.0, 0.0]
    xs, ys, xe, ye, cc, xp = W, H, 0, 0, 0, 0
    for j in range(m):
        cc += counts[j]
        t = cc - j % 2
        y, x = t % H, t // H
        if j % 2 == 0:
            xp = x
        elif xp < x:
            ys, ye = 0, H - 1
        xs, xe, ys, ye = min(xs, x), max(xe, x), min(ys, y), max(ye, y)
    return [float(xs), float(ys), float(xe - xs + 1), float(ye - ys + 1)]


def encode_masks(masks):
    """[n, H, W] masks -> list of {"size": [H, W], "counts": bytes}, the output of pycocotools.mask.encode on the
    Fortran-ordered [H, W, n] uint8 stack."""
    masks = np.asarray(masks)
    H, W = masks.shape[-2:]
    return [{"size": [int(H), int(W)], "counts": to_string(encode(m))} for m in masks.reshape(-1, H, W)]
