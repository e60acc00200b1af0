"""TEST INFRASTRUCTURE — numpy restatement of the reference's DAVIS evaluation loop (psalm/eval/eval_davis.py:388-480),
driven by `PSALMForDAVISEval.eval_video` results: the per-object query pick, `fuse_davis_mask`, the memory check and the
memory update with detectron2's `ResizeTransform.apply_segmentation` + FixedSizeCrop padding.  The colour image and
the PNG writing (:484-498) are left out.  Used by the tests and by tools/bench_video.py as "what a user writes today"."""
import numpy as np

TOPK = 10   # eval_davis.py:446


def pick_objects(scores_qk):
    """eval_davis.py:436-453.  scores_qk [Q,K] (`output['instances'].scores`) -> (pick [K] int64, pick_score [K] fp32).
    The top 10 queries of each object in score order are tried; the first one no earlier object took is picked.  When
    all 10 are taken, `pick_idx` / `pick_score` keep the previous object's values (the reference's loop variables).
    Ties go to the lower query index (torch's CPU `topk` leaves their order undefined)."""
    scores = np.asarray(scores_qk, dtype=np.float32).T          # :436 .transpose(1, 0)
    prev_idx = []
    picks, pick_scores = [], []
    pick_idx, pick_score = None, None
    for i in range(len(scores)):
        cur = scores[i]
        idx = np.lexsort((np.arange(len(cur)), -cur))[:TOPK]    # descending score, ascending index on ties
        for j in range(TOPK):
            if idx[j] not in prev_idx:
                prev_idx.append(idx[j])
                pick_idx, pick_score = int(idx[j]), cur[idx[j]]
                break
        picks.append(pick_idx)
        pick_scores.append(pick_score)
    return np.array(picks, dtype=np.int64), np.array(pick_scores, dtype=np.float32)


def fuse_davis_mask(mask_list, fill_number_list):
    """eval_davis.py:337-342."""
    fused_mask = np.zeros_like(mask_list[0])
    for mask, fill_number in zip(mask_list, fill_number_list):
        fused_mask[mask == 1] = int(fill_number)
    return fused_mask


def memory_correct(mask_list):
    """eval_davis.py:464-473: False when two different objects overlap with IoU > 0.4 (0 / 0 is NaN: no failure)."""
    flag = True
    with np.errstate(divide="ignore", invalid="ignore"):
        for i in range(len(mask_list)):
            for j in range(len(mask_list)):
                if i != j:
                    intersection = np.logical_and(mask_list[i], mask_list[j])
                    union = np.logical_or(mask_list[i], mask_list[j])
                    if np.sum(intersection) / np.sum(union) > 0.4:
                        flag = False
    return flag


def _pil_nearest_index(in_size, out_size):
    """Pillow's Image.resize(NEAREST) source index per output pixel (Geometry.c ImagingScaleAffine: start at scale / 2,
    add the scale once per pixel in double, truncate; -1 = left unset)."""
    scale = in_size / out_size
    out, xo = [], scale * 0.5
    for _ in range(out_size):
        xin = -1 if xo < 0 else int(xo)
        out.append(xin if xin < in_size else -1)
        xo += scale
    return np.array(out, dtype=np.int64)


def apply_segmentation(mask, resized_hw, padded_hw):
    """detectron2 ResizeTransform.apply_segmentation (uint8 -> Pillow NEAREST to `resized_hw`) then FixedSizeCrop's
    PadTransform (zeros at the bottom / right, seg_pad_value=0 in the reference mappers) to `padded_hw`."""
    (oh, ow), (Hp, Wp) = resized_hw, padded_hw
    r, c = _pil_nearest_index(mask.shape[0], oh), _pil_nearest_index(mask.shape[1], ow)
    out = np.zeros((Hp, Wp), dtype=mask.dtype)
    res = mask[np.clip(r, 0, None)][:, np.clip(c, 0, None)]
    res[r < 0] = 0
    res[:, c < 0] = 0
    out[:oh, :ow] = res
    return out


class DavisLoop:
    """The loop state of one clip (eval_davis.py:379-383, :392-480): prev_mask_list, prev_fill_number_list, prev_image
    and prev_transformer (here the resized and padded sizes of the memory frame)."""

    def __init__(self, first_image, first_masks, fill_numbers, with_memory=True):
        self.first_image, self.first_masks = first_image, np.asarray(first_masks, dtype=bool)
        self.fills = [int(f) for f in fill_numbers]
        self.with_memory = with_memory
        self.prev_mask_list, self.prev_fill_number_list = [], []
        self.prev_image, self.prev_sizes = None, None

    def inputs(self):
        """(vp_images, vp_region_masks bool [K,Hp,Wp], vp_fill_number) for the next eval_video call (:401-419)."""
        if self.with_memory and len(self.prev_mask_list) != 0 and len(self.fills) == len(self.prev_fill_number_list):
            masks = np.stack([apply_segmentation(m, *self.prev_sizes) for m in self.prev_mask_list])
            return self.prev_image, masks.astype(bool), list(self.prev_fill_number_list)
        return self.first_image, self.first_masks, list(self.fills)

    def update(self, output, fill_numbers, image, resized_hw, padded_hw):
        """:433-480 on `output` = eval_video(...)[0].  Returns dict(labels uint8 [H,W], pick, score, memory_updated)."""
        pred_mask = output["instances"].pred_masks.cpu().numpy()
        scores = output["instances"].scores.cpu().numpy()           # [Q,K]
        assert scores.shape[1] == len(fill_numbers)
        pick, score = pick_objects(scores)
        pred_mask_list = [pred_mask[p].astype(np.uint8) for p in pick]
        labels = fuse_davis_mask(pred_mask_list, fill_numbers)
        updated = False
        if self.with_memory and memory_correct(pred_mask_list):
            self.prev_mask_list, self.prev_fill_number_list = pred_mask_list, list(fill_numbers)
            self.prev_image, self.prev_sizes = image, (resized_hw, padded_hw)
            updated = True
        return dict(labels=labels, pick=pick, score=score, memory_updated=updated)
