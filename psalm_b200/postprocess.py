"""Post-processing of eval_seg (reference language_model/llava_phi.py:1395-1472 and the task heads
:308-447), on the GPU.  detectron2's `sem_seg_postprocess` / `ImageList.from_tensors` (third-party,
un-vendored, version unpinned upstream) are restated: crop to the un-padded box, bilinear resize.

Panoptic merging: the reference loops over kept segments in Python with several `.item()` syncs per
segment (:356-384).  Here the per-segment areas are three batched reductions, ONE small D2H copy
brings (keep, class, areas) to the host, the sequential merge rule (stuff classes share an id, overlap
threshold 0.8) runs on <= 100 integers, and a lookup table maps the arg-max map to segment ids on the
device."""
import numpy as np
import torch
import torch.nn.functional as F

from .structures import Boxes, Instances


def unpadded_box(padding_mask):
    """llava_phi.py:1418-1423: bounding box of ~padding_mask (host side, like the reference)."""
    pm = padding_mask.cpu().numpy() if isinstance(padding_mask, torch.Tensor) else np.asarray(padding_mask)
    keep = ~pm.astype(bool)
    # extent of the rows / columns that hold any un-padded pixel (same box as nonzero(): min / max index per axis,
    # without materialising the 10^6-entry index arrays: 0.2 ms instead of 6 ms per 1024^2 mask)
    rows, cols = np.flatnonzero(keep.any(axis=1)), np.flatnonzero(keep.any(axis=0))
    return int(rows[-1] - rows[0] + 1), int(cols[-1] - cols[0] + 1)


def sem_seg_postprocess(result, img_size, out_h, out_w):
    result = result[:, : img_size[0], : img_size[1]].unsqueeze(0)
    if result.shape[-2:] == (out_h, out_w):
        return result[0]
    return F.interpolate(result, size=(out_h, out_w), mode="bilinear", align_corners=False)[0]


def semantic_inference(cls, mask_pred, sig=None, tf32=False):
    """softmax(cls)[:, :-1]^T . sigmoid(mask)  (llava_phi.py:402-406) as one library GEMM
    (TF32 tensor cores when the model runs in 16-bit storage, exact fp32 for parity runs)."""
    probs = F.softmax(cls.float(), dim=-1)[:, :-1]
    Q, H, W = mask_pred.shape
    if sig is None:
        sig = mask_pred.float().sigmoid()
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = bool(tf32)
    try:
        out = torch.matmul(probs.t(), sig.view(Q, H * W)).view(-1, H, W)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    return out


def query_mask_scores(mask_pred, sig=None):
    """Per-QUERY mask score  sum(sigmoid * [logit > 0]) / (sum([logit > 0]) + 1e-6)  (llava_phi.py:441-443).
    It depends only on the query, so it is computed once for the 100 queries instead of once per
    selected (query, class) pair."""
    if sig is None:
        sig = mask_pred.float().sigmoid()
    pos = mask_pred > 0
    num = torch.where(pos, sig, torch.zeros((), dtype=sig.dtype, device=sig.device)).flatten(1).sum(1)
    return num / (pos.flatten(1).sum(1).float() + 1e-6)


def instance_inference(cls, mask_pred, topk, is_thing_list=None, panoptic_on=False, sig=None):
    """llava_phi.py:407-447 (topk(sorted=False): order is implementation defined; compare as sets)."""
    scores = F.softmax(cls.float(), dim=-1)[:, :-1]
    nq, nc = scores.shape
    s, idx = scores.flatten(0, 1).topk(topk, sorted=False)
    lab = idx % nc
    qi = idx // nc
    if panoptic_on:
        thing = torch.as_tensor([bool(t) for t in is_thing_list], device=cls.device)
        keep = thing[lab]
        s, lab, qi = s[keep], lab[keep], qi[keep]
    ms = query_mask_scores(mask_pred, sig)[qi]
    r = Instances(tuple(mask_pred.shape[-2:]))
    r.pred_masks = (mask_pred.index_select(0, qi) > 0).float()
    r.pred_boxes = Boxes(torch.zeros(qi.shape[0], 4))
    r.scores = s * ms
    r.pred_classes = lab
    r.query_index = qi
    return r


def seg_instance_inference(SEG_cls, mask_pred, topk, sig=None):
    """llava_phi.py:308-324 (referring segmentation)."""
    scores = torch.sigmoid(SEG_cls.float())
    s, idx = scores.flatten(0, 1).topk(topk, sorted=False)
    ms = query_mask_scores(mask_pred, sig)[idx]
    r = Instances(tuple(mask_pred.shape[-2:]))
    r.pred_masks = (mask_pred.index_select(0, idx) > 0).float()
    r.pred_boxes = Boxes(torch.zeros(idx.shape[0], 4))
    r.scores = s * ms
    r.query_index = idx
    return r


def region_inference(region_cls, mask_pred, sig=None):
    """llava_phi.py:387-400 (region prompts): region_cls [K,Q] -> Instances(pred_masks [Q,H,W], scores [Q,K])."""
    ms = query_mask_scores(mask_pred, sig)
    r = Instances(tuple(mask_pred.shape[-2:]))
    r.pred_masks = (mask_pred > 0).float()
    r.pred_boxes = Boxes(torch.zeros(mask_pred.shape[0], 4))
    r.scores = (torch.sigmoid(region_cls.float()) * ms[None, :]).transpose(1, 0)
    return r


def panoptic_inference(cls, mask_pred, is_thing_list, obj_thr=0.8, ovl_thr=0.8, sig=None):
    """llava_phi.py:325-386 -> (panoptic_seg int32 [H,W], segments_info list)."""
    scores, labels = F.softmax(cls.float(), dim=-1).max(-1)
    nc = cls.shape[-1] - 1
    Q, H, W = mask_pred.shape
    if sig is None:
        sig = mask_pred.float().sigmoid()
    keep = labels.ne(nc) & (scores > obj_thr)
    # argmax over kept queries only: non-kept rows evaluate to -1 (< any kept score * sigmoid >= 0)
    wq = torch.where(keep, scores, torch.zeros_like(scores)).view(Q, 1, 1)
    neg = (keep.float() - 1.0).view(Q, 1, 1)
    ids = torch.addcmul(neg, sig, wq).argmax(0).view(-1)                  # [H*W] query index
    in_mask = mask_pred.view(Q, -1).gather(0, ids.view(1, -1)).view(-1) >= 0   # sigmoid >= 0.5 at the winner
    area = torch.bincount(ids, minlength=Q)
    inter = torch.bincount(ids, weights=in_mask.float(), minlength=Q).long()
    orig = (mask_pred >= 0).flatten(1).sum(1)
    host = torch.stack([keep.long(), labels.long(), area, orig, inter], 0).cpu().numpy()   # the one D2H copy
    if host[0].sum() == 0:
        return torch.zeros((H, W), dtype=torch.int32, device=cls.device), []
    seg_of_query, info = panoptic_merge(host, is_thing_list, ovl_thr)
    lut = torch.from_numpy(seg_of_query).to(cls.device)
    pan = torch.where(in_mask, lut[ids], torch.zeros((), dtype=torch.int32, device=cls.device))
    return pan.view(H, W).to(torch.int32), info


def panoptic_merge(host, is_thing_list, ovl_thr):
    """The reference's sequential merge rule (llava_phi.py:355-384) on the per-query integers host [5, Q] (rows: keep,
    class, area, original area, intersection): stuff classes share one segment id, a query whose visible area is below
    `ovl_thr` of its own mask is dropped.  Returns (seg_of_query int32 [Q], 0 = no segment; segments_info)."""
    Q = host.shape[1]
    seg_of_query = np.zeros(Q, np.int32)
    info, stuff, cur = [], {}, 0
    for q in range(Q):
        if not host[0, q]:
            continue
        pc, a, o, it = int(host[1, q]), int(host[2, q]), int(host[3, q]), int(host[4, q])
        if a > 0 and o > 0 and it > 0:
            if a / o < ovl_thr:
                continue
            isthing = bool(is_thing_list[pc])
            if not isthing:
                if pc in stuff:
                    seg_of_query[q] = stuff[pc]
                    continue
                stuff[pc] = cur + 1
            cur += 1
            seg_of_query[q] = cur
            info.append(dict(id=cur, isthing=isthing, category_id=pc))
    return seg_of_query, info


_THING_CACHE = {}


def thing_tensor(is_thing_list, device):
    """Boolean `is_thing` lookup table on the device, cached by content (built once per class vocabulary)."""
    key = (tuple(bool(t) for t in is_thing_list), str(device))
    if key not in _THING_CACHE:
        _THING_CACHE[key] = torch.tensor(key[0], dtype=torch.bool, device=device)
    return _THING_CACHE[key]


# Limits of the fused task-head kernel (csrc/postproc.cu): at most 104 queries and 144 classes; its class-probability
# operand `probsT` is fp16 [144, 112], zero padded (queries padded to 112).
FUSED_MAX_QUERIES, FUSED_MAX_CLASSES, FUSED_PADDED_QUERIES = 104, 144, 112


def fused_device_batch(kernels, logits, sizes, cls=None, SEG_cls=None, thing=None, semantic_on=False, instance_on=False,
                       panoptic_on=False, referring_on=False, topk=100, obj_thr=0.8, crops=None):
    """Device part of the fused task heads for a batch (no host synchronisation, CUDA-graph capturable): the small
    [Q, n_cls] algebra (softmax, arg-max, top-k, stable partition of the kept slots) runs ONCE on [B, ...] tensors
    instead of once per image (~25 tiny launches per image, among them a 57 us single-block top-k), then one fused kernel
    (csrc/postproc.cu) per image on its LOW-RESOLUTION mask logits.  logits [B,Q,H4,W4]; sizes / crops: per image (H, W)
    and None | (Hp, Wp, oh, ow).  Returns the list of per-image dicts `fused_host` consumes; each holds `hostvec`, the
    one vector its host part needs."""
    B, Q = logits.shape[:2]
    dev = logits.device
    probsT = wq = negq = slots = None
    ncls = 0
    if cls is not None:
        probs_full = F.softmax(cls.float(), dim=-1)          # [B,Q,C+1]
        probs = probs_full[..., :-1]
        ncls = probs.shape[-1]
    if semantic_on:
        probsT = torch.zeros((B, FUSED_MAX_CLASSES, FUSED_PADDED_QUERIES), dtype=torch.float16, device=dev)
        probsT[:, :ncls, :Q] = probs.transpose(1, 2).to(torch.float16)
    if panoptic_on:
        scores, labels = probs_full.max(-1)
        keep = labels.ne(ncls) & (scores > obj_thr)
        wq = torch.where(keep, scores, torch.zeros_like(scores)).contiguous()
        negq = (keep.float() - 1.0).contiguous()
    s = lab = qi = keep_i = None
    if instance_on:
        s, idx = probs.flatten(1, 2).topk(topk, dim=1, sorted=False)
        lab, qi = idx % ncls, idx // ncls
        if panoptic_on:
            keep_i = thing[lab]
            order = torch.sort((~keep_i).to(torch.uint8), dim=1, stable=True).indices      # kept slots first
            s, lab, qi, keep_i = (t.gather(1, order) for t in (s, lab, qi, keep_i))
        else:
            keep_i = torch.ones_like(qi, dtype=torch.bool)
        slots = torch.where(keep_i, qi, torch.full_like(qi, -1)).to(torch.int32).contiguous()
    elif referring_on:
        s, qi = torch.sigmoid(SEG_cls.float()).flatten(1, 2).topk(topk, dim=1, sorted=False)
        keep_i = torch.ones_like(qi, dtype=torch.bool)
        slots = qi.to(torch.int32).contiguous()
    ks = []
    for b in range(B):
        H, W = sizes[b]
        ks.append(kernels.postproc_fused(logits[b].contiguous(), H, W, probsT[b] if probsT is not None else None,
                                         wq[b] if wq is not None else None, negq[b] if negq is not None else None,
                                         slots[b] if slots is not None else None, ncls,
                                         crop=crops[b] if crops is not None else None))
    st = torch.stack([k["stats"] for k in ks])               # [B,Q,5]
    rows = []
    inst_scores = None
    if slots is not None:
        rows.append(keep_i.sum(1, keepdim=True).float())
        inst_scores = s * (st[..., 1] / (st[..., 0] + 1e-6)).gather(1, qi)       # class score x per-query mask score
    if panoptic_on:
        rows += [keep.float(), labels.float(), st[..., 3], st[..., 2], st[..., 4]]
    hostvec = torch.cat(rows, 1).contiguous() if rows else None
    out = []
    for b in range(B):
        H, W = sizes[b]
        d = dict(Q=Q, H=H, W=W, sem_seg=ks[b]["sem_seg"], inst_masks=ks[b]["inst_masks"], ids=ks[b]["ids"],
                 in_mask=ks[b]["in_mask"], lab=lab[b] if lab is not None else None, qi=qi[b] if qi is not None else None,
                 hostvec=hostvec[b] if hostvec is not None else None, has_inst=slots is not None, has_pan=bool(panoptic_on),
                 has_sem=bool(semantic_on))
        if inst_scores is not None:
            d["inst_scores"] = inst_scores[b]
        out.append(d)
    return out


def fused_host(d, is_thing_list=None, ovl_thr=0.8, host=None):
    """Host part: the ONE D2H copy, the sequential panoptic merge rule on <= Q integers
    (llava_phi.py:355-384) and the final id lookup."""
    Q, H, W = d["Q"], d["H"], d["W"]
    r = {}
    if d["has_sem"]:
        r["sem_seg"] = d["sem_seg"]
    if host is None:   # (else: already copied into pinned memory behind the pass, PSALM.eval_seg_async)
        host = d["hostvec"].cpu().numpy() if d["hostvec"] is not None else None    # the one D2H copy
    pos = 0
    if d["has_inst"]:
        n_inst = int(host[0])
        pos = 1
        inst = Instances((H, W))
        inst.pred_masks = d["inst_masks"][:n_inst]
        inst.pred_boxes = Boxes(torch.zeros(n_inst, 4))
        inst.scores = d["inst_scores"][:n_inst]
        if d["lab"] is not None:
            inst.pred_classes = d["lab"][:n_inst]
        inst.query_index = d["qi"][:n_inst]
        r["instances"] = inst
    if d["has_pan"]:
        dev = d["ids"].device
        hk = host[pos:].reshape(5, Q)
        if hk[0].sum() == 0:
            pan, info = torch.zeros((H, W), dtype=torch.int32, device=dev), []
        else:
            seg_of_query, info = panoptic_merge(hk, is_thing_list, ovl_thr)
            lut = torch.from_numpy(seg_of_query).to(dev)
            pan = torch.where(d["in_mask"].bool(), lut[d["ids"].long()], torch.zeros((), dtype=torch.int32, device=dev))
        r["panoptic_seg"] = (pan.to(torch.int32), info)
    return r
