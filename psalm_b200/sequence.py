"""Sequence assembly for the LLM prefill — host logic of the hot path.

Restates `PSALM.prepare_inputs_labels_for_multimodal` / `concat_image_seg_cls_embeds`
(reference language_model/llava_phi.py:767-971, 581-766) and the embedding-extraction helpers
`get_seg_query` (:1299-1316), `get_class_name_embedding` (:552-565), `get_SEG_embedding` (:972-978).

The reference walks every token id in Python with `.item()` (llava_phi.py:614-623) and launches
~270 tiny kernels for class-name pooling.  Here the prompt is turned ONCE, on the host, into an index
*plan* (numpy, loops only over the ~140 sentinel ids); the device side is then four library calls:
one embedding gather, two row scatters (image tokens, seg queries) and one pooling matmul.
Sentinel ids (psalm/constants.py:8-12): <image> -200, <seg> -201, <cls> -202, <region> -203, <refer> -204.
"""
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

IMAGE_TOKEN_INDEX = -200
SEG_TOKEN_INDEX = -201
CLS_TOKEN_INDEX = -202
REGION_TOKEN_INDEX = -203
REFER_TOKEN_INDEX = -204


@dataclass
class SequencePlan:
    B: int
    T: int
    tok_ids: torch.Tensor            # [B,T] int64  token id to embed (0 where the row comes from elsewhere)
    img_pos: torch.Tensor            # [B*n_img] int64 flat row index (b*T + t) of every image token
    seg_pos: torch.Tensor            # [B*n_q]  int64 flat row index of every seg-query token
    pad_pos: Optional[torch.Tensor]  # flat rows that are right padding (zero embeddings), or None
    attention_mask: torch.Tensor     # [B,T] bool
    any_padding: bool
    cls_pool: Optional[torch.Tensor]   # [B,n_cls,T] fp32 averaging matrix (rows sum to 1), or None
    refer_pool: Optional[torch.Tensor]  # [B,1,T] fp32, or None
    n_img: int
    n_q: int
    region_pos: Optional[torch.Tensor] = None   # [R] int64 flat rows of the <region> tokens (sample-major, prompt order)
    region_counts: Optional[tuple] = None        # regions per sample
    region_points: Optional[torch.Tensor] = None  # [R,P,2] fp32 sample points (y, x) in [0,1], set by the caller
    region_image: Optional[torch.Tensor] = None   # [R] int32 image index of every region
    vp_images: Optional[torch.Tensor] = None      # [B,3,H,W] visual-prompt frames the regions are pooled from (DAVIS variant)

    def to(self, device):
        mv = lambda t: None if t is None else t.to(device, non_blocking=True)  # noqa: E731
        return SequencePlan(self.B, self.T, mv(self.tok_ids), mv(self.img_pos), mv(self.seg_pos), mv(self.pad_pos),
                            mv(self.attention_mask), self.any_padding, mv(self.cls_pool), mv(self.refer_pool),
                            self.n_img, self.n_q, mv(self.region_pos), self.region_counts, mv(self.region_points),
                            mv(self.region_image), mv(self.vp_images))


def build_plan(input_ids, attention_mask, n_img, n_q, class_name_ids=None, cls_indices=None,
               class_name_embedding_indices=None, token_refer_id=None, refer_embedding_indices=None, suffix=False):
    """All arguments are HOST tensors in the reference's input contract (train_datasets.py:186-234).
    suffix=True: the rows are prompt suffixes behind a shared prefix that holds the <image> (split_prompts); they carry
    no <image> sentinel, and a class list may be shorter than the longest of the batch (its extra pooling rows are 0)."""
    ids_all = input_ids.cpu().numpy()
    B, T0 = ids_all.shape
    am_all = np.ones((B, T0), bool) if attention_mask is None else attention_mask.cpu().numpy().astype(bool)
    has_region = bool((ids_all == REGION_TOKEN_INDEX).any())
    rows = []
    for b in range(B):
        ids = ids_all[b]
        assert (ids == IMAGE_TOKEN_INDEX).sum() == (0 if suffix else 1), "not supporting multi image index"   # llava_phi.py:588
        assert (ids == SEG_TOKEN_INDEX).sum() == 1, "not supporting multi seg index"       # llava_phi.py:589
        names = None
        if class_name_ids is not None:  # embed_class_ids, llava_phi.py:566-575
            cn = class_name_ids[b].cpu().numpy()
            ci = cls_indices[b].cpu().numpy()
            names = []
            prev = None
            for u in ci:  # unique_consecutive, then drop the -1 padding
                if u != prev:
                    prev = u
                    if u >= 0:
                        names.append(cn[ci == u])
            assert (ids == CLS_TOKEN_INDEX).sum() == len(names), \
                "the number of <cls> tokens and class_embed needs to be same"               # llava_phi.py:590-591
        refer = token_refer_id[b].cpu().numpy() if token_refer_id is not None else None
        cei = class_name_embedding_indices[b].cpu().numpy() if class_name_embedding_indices is not None else None
        rei = refer_embedding_indices[b].cpu().numpy() if refer_embedding_indices is not None else None
        tok, kind, cidx, ridx = [], [], [], []   # kind: 1 text, 2 image, 3 seg, 4 region feature
        special = np.nonzero(ids < 0)[0]
        prev_end = 0
        cls_i = 0

        def text(lo, hi):
            if hi > lo:
                tok.append(ids[lo:hi]); kind.append(np.full(hi - lo, 1))
                cidx.append(cei[lo:hi] if cei is not None else np.zeros(hi - lo, np.int64))
                ridx.append(rei[lo:hi] if rei is not None else np.zeros(hi - lo, np.int64))

        for sp in special:
            text(prev_end, sp)
            t = ids[sp]
            if t == IMAGE_TOKEN_INDEX:
                n, k, tk, cv, rv = n_img, 2, np.zeros(n_img, np.int64), 0, 0
            elif t == SEG_TOKEN_INDEX:
                n, k, tk, cv, rv = n_q, 3, np.zeros(n_q, np.int64), 0, 0
            elif t == CLS_TOKEN_INDEX:
                tk = names[cls_i]
                cls_i += 1
                n, k, cv, rv = len(tk), 1, cls_i, 0   # 1-based running class counter (llava_phi.py:671-673)
            elif t == REFER_TOKEN_INDEX:
                tk = refer
                n, k, cv, rv = len(tk), 1, 0, 1
            elif t == REGION_TOKEN_INDEX:   # one row per region, filled with its pooled feature (llava_phi.py:684-703)
                n, k, tk, cv, rv = 1, 4, np.zeros(1, np.int64), 0, 0
            else:
                raise ValueError("unknown sentinel id %d" % t)
            tok.append(tk); kind.append(np.full(n, k)); cidx.append(np.full(n, cv)); ridx.append(np.full(n, rv))
            prev_end = sp + 1
        text(prev_end, T0)
        tok, kind, cidx, ridx = map(np.concatenate, (tok, kind, cidx, ridx))
        # attention mask: inserted tokens attendable, then the caller's mask (llava_phi.py:935-949, 964-969)
        am = np.concatenate([np.ones(len(tok) - T0, bool), am_all[b]])
        rows.append((tok, kind, cidx, ridx, am))
    T = max(len(r[0]) for r in rows)
    tok_ids = np.zeros((B, T), np.int64)
    attn = np.zeros((B, T), bool)
    cls_idx = np.zeros((B, T), np.int64)
    ref_idx = np.zeros((B, T), np.int64)
    img_pos, seg_pos, pad_pos, region_pos, region_counts = [], [], [], [], []
    for b, (tok, kind, cidx, ridx, am) in enumerate(rows):
        n = len(tok)
        tok_ids[b, :n] = np.where(kind == 1, tok, 0)
        attn[b, :n] = am
        cls_idx[b, :n] = cidx
        ref_idx[b, :n] = ridx
        img_pos.append(b * T + np.nonzero(kind == 2)[0])
        seg_pos.append(b * T + np.nonzero(kind == 3)[0])
        region_pos.append(b * T + np.nonzero(kind == 4)[0])
        region_counts.append(int((kind == 4).sum()))
        pad_pos.append(b * T + np.arange(n, T))
    pad_pos = np.concatenate(pad_pos)
    cls_pool = refer_pool = None
    if class_name_embedding_indices is not None:
        ncls = int(cls_idx.max())
        cls_pool = np.zeros((B, ncls, T), np.float32)
        for b in range(B):
            for c in range(1, ncls + 1):
                m = cls_idx[b] == c
                if suffix and not m.any():   # a shorter class list than the batch's longest
                    continue
                assert m.any(), "class %d has no tokens in sample %d" % (c, b)
                cls_pool[b, c - 1, m] = 1.0 / m.sum()   # AdaptiveAvgPool1d(1), llava_phi.py:561-563
    if refer_embedding_indices is not None:
        refer_pool = np.zeros((B, 1, T), np.float32)
        for b in range(B):
            m = ref_idx[b] != 0
            refer_pool[b, 0, m] = 1.0 / m.sum()
    any_padding = bool((~attn).any())
    ft = torch.from_numpy
    return SequencePlan(B, T, ft(tok_ids), ft(np.concatenate(img_pos)), ft(np.concatenate(seg_pos)),
                        ft(pad_pos) if len(pad_pos) else None, ft(attn), any_padding,
                        ft(cls_pool) if cls_pool is not None else None,
                        ft(refer_pool) if refer_pool is not None else None, n_img, n_q,
                        ft(np.concatenate(region_pos)) if has_region else None,
                        tuple(region_counts) if has_region else None)


def materialize_embeds(plan, embed_tokens, image_tokens, seg_query, region_features=None):
    """plan on device; embed_tokens [V,C]; image_tokens [B,n_img,C]; seg_query [n_q,C]; region_features [R,C] (one
    row per <region> token, plan.region_pos order) -> inputs_embeds [B,T,C]."""
    B, T = plan.B, plan.T
    C = embed_tokens.shape[1]
    flat = embed_tokens.index_select(0, plan.tok_ids.view(-1))
    flat.index_copy_(0, plan.img_pos, image_tokens.reshape(-1, C).to(flat.dtype))
    flat.index_copy_(0, plan.seg_pos, seg_query.to(flat.dtype).repeat(B, 1))
    if plan.region_pos is not None:
        flat.index_copy_(0, plan.region_pos, region_features.to(flat.dtype))
    if plan.pad_pos is not None:
        flat.index_fill_(0, plan.pad_pos, 0)   # right padding rows are zeros (llava_phi.py:878-883)
    return flat.view(B, T, C)


def gather_seg_query(plan, hidden):
    """hidden [B,T,C] -> [B,n_q,C]  (get_seg_query, llava_phi.py:1299-1316)."""
    return hidden.reshape(plan.B * plan.T, -1).index_select(0, plan.seg_pos).view(plan.B, plan.n_q, -1)


def pool(pool_matrix, hidden):
    """[B,n,T] averaging matrix x [B,T,C] -> [B,n,C] (class-name / [SEG] mean pooling)."""
    return torch.bmm(pool_matrix.to(hidden.dtype), hidden)


def gather_region_rows(plan, hidden):
    """hidden [B,T,C] -> [R,C] hidden states at the <region> positions (get_region_embedding, llava_phi.py:302-307)."""
    return hidden.reshape(plan.B * plan.T, -1).index_select(0, plan.region_pos)


# ---- several prompts against one image: shared prefix + per-prompt suffixes ---------------------------------------
OUTPUT_SENTINELS = (SEG_TOKEN_INDEX, CLS_TOKEN_INDEX, REFER_TOKEN_INDEX, REGION_TOKEN_INDEX)
PROMPT_KEYS = ("input_ids", "attention_mask", "token_refer_id", "refer_embedding_indices", "class_name_ids", "cls_indices",
               "class_name_embedding_indices")


@dataclass
class PromptSplit:
    prefix_ids: np.ndarray      # [L] int64 input ids of the shared prefix (holds the <image> sentinel)
    P: int                      # rows of the prefix after the <image> expansion
    tok_ids: torch.Tensor       # [1,P] int64 token id of every prefix row (0 on image rows)
    img_pos: torch.Tensor       # [n_img] int64 prefix rows of the image tokens
    suffix: SequencePlan        # [K, Ts] plan of the remaining tokens of every prompt (right padded)
    n_classes: tuple            # classes of every prompt (0 without a class list)


def _row(t, name):
    """One prompt's tensor: [T] or [1, T] (a list / tuple of one tensor for token_refer_id) -> host 1-D tensor."""
    if t is None:
        return None
    if isinstance(t, (list, tuple)):
        if len(t) != 1:
            raise ValueError("%s: one prompt per dict (got %d rows)" % (name, len(t)))
        t = t[0]
    t = torch.as_tensor(t).cpu()
    if t.dim() == 2:
        if t.shape[0] != 1:
            raise ValueError("%s: one prompt per dict (got %d rows)" % (name, t.shape[0]))
        t = t[0]
    return t


def split_prompts(prompts, n_img, n_q):
    """Cut K prompts of one image into the shared prefix and K suffixes (input_ids space).  The prefix is the longest
    common token prefix of the prompts, truncated at the first position that feeds an output (a <seg>, <cls>, <refer> or
    <region> sentinel, or a non-zero class-name / refer embedding index).  It must hold the <image> sentinel and no masked
    position.  <region> prompts need their regions as `visual_prompts` (one (kind, source) pair per <region> token, see
    ImageSession.eval_seg); the suffixes then carry region_pos / region_counts.  Raises ValueError (or
    NotImplementedError for <region> prompts without visual_prompts) instead of falling back."""
    if not prompts:
        raise ValueError("no prompts")
    if len({"visual_prompts" in p for p in prompts}) > 1:
        raise ValueError("prompts of one call must all have or all lack visual_prompts")
    rows = []
    for k, p in enumerate(prompts):
        unknown = set(p) - set(PROMPT_KEYS) - {"is_thing_list", "visual_prompts"}
        if unknown:
            raise ValueError("prompt %d: unknown keys %s" % (k, sorted(unknown)))
        r = {n: _row(p.get(n), n) for n in PROMPT_KEYS if n not in ("class_name_ids", "cls_indices", "token_refer_id")}
        r["ids"] = r.pop("input_ids").numpy().astype(np.int64)
        n_regions = int((r["ids"] == REGION_TOKEN_INDEX).sum())
        if n_regions and "visual_prompts" not in p:
            raise NotImplementedError("<region> prompts of a session need their regions as visual_prompts (the "
                                      "per-image region_masks of eval_seg are not read by sessions)")
        if "visual_prompts" in p and len(p["visual_prompts"]) != n_regions:
            raise ValueError("prompt %d: %d visual prompts for %d <region> tokens" % (k, len(p["visual_prompts"]),
                                                                                    n_regions))
        T0 = len(r["ids"])
        r["am"] = np.ones(T0, bool) if r["attention_mask"] is None else r["attention_mask"].numpy().astype(bool)
        r["cei"] = None if r["class_name_embedding_indices"] is None else r["class_name_embedding_indices"].numpy()
        r["rei"] = None if r["refer_embedding_indices"] is None else r["refer_embedding_indices"].numpy()
        for n in ("class_name_ids", "cls_indices", "token_refer_id"):
            r[n] = _row(p.get(n), n)
        rows.append(r)
    for n in ("class_name_ids", "token_refer_id", "cei", "rei"):
        if len({rows[k][n] is None for k in range(len(rows))}) > 1:
            raise ValueError("prompts of one call must all have or all lack %s" % n)
    ids0 = rows[0]["ids"]
    L = min(len(r["ids"]) for r in rows)
    for r in rows[1:]:
        neq = np.nonzero(r["ids"][:L] != ids0[:L])[0]
        if len(neq):
            L = int(neq[0])
    feeds = np.isin(ids0[:L], OUTPUT_SENTINELS)
    for r in rows:
        for n in ("cei", "rei"):
            if r[n] is not None:
                feeds |= r[n][:L] != 0
    if feeds.any():
        L = int(np.nonzero(feeds)[0][0])
    img = np.nonzero(ids0[:L] == IMAGE_TOKEN_INDEX)[0]
    if len(img) != 1:
        raise ValueError("the shared prefix of the prompts (%d tokens) does not contain the <image> sentinel: the prompts "
                         "differ, or feed an output, before <image>" % L)
    for k, r in enumerate(rows):
        if not r["am"][:L].all():
            raise ValueError("prompt %d has a masked position inside the shared prefix (first %d tokens)" % (k, L))
    i0 = int(img[0])
    P = L - 1 + n_img
    tok = np.concatenate([ids0[:i0], np.zeros(n_img, np.int64), ids0[i0 + 1:L]])
    Ts0 = max(len(r["ids"]) - L for r in rows)
    K = len(rows)
    ids = np.zeros((K, Ts0), np.int64)
    am = np.zeros((K, Ts0), bool)
    cei = np.zeros((K, Ts0), np.int64) if rows[0]["cei"] is not None else None
    rei = np.zeros((K, Ts0), np.int64) if rows[0]["rei"] is not None else None
    for k, r in enumerate(rows):
        n = len(r["ids"]) - L
        ids[k, :n], am[k, :n] = r["ids"][L:], r["am"][L:]
        if cei is not None:
            cei[k, :n] = r["cei"][L:]
        if rei is not None:
            rei[k, :n] = r["rei"][L:]
    ft = torch.from_numpy
    has_cls = rows[0]["class_name_ids"] is not None
    plan = build_plan(ft(ids), ft(am), n_img, n_q,
                      [r["class_name_ids"] for r in rows] if has_cls else None,
                      [r["cls_indices"] for r in rows] if has_cls else None,
                      ft(cei) if cei is not None else None,
                      [r["token_refer_id"] for r in rows] if rows[0]["token_refer_id"] is not None else None,
                      ft(rei) if rei is not None else None, suffix=True)
    n_classes = tuple(int((ids[k] == CLS_TOKEN_INDEX).sum()) for k in range(K))
    return PromptSplit(ids0[:L].copy(), P, ft(tok).view(1, P), ft(i0 + np.arange(n_img, dtype=np.int64)), plan, n_classes)


def prefix_embeds(split, embed_tokens, image_tokens):
    """Shared prefix rows [1,P,C]: token embeddings with the projector tokens image_tokens [1,n_img,C] at the image rows."""
    C = embed_tokens.shape[1]
    flat = embed_tokens.index_select(0, split.tok_ids.view(-1))
    flat.index_copy_(0, split.img_pos, image_tokens.reshape(-1, C).to(flat.dtype))
    return flat.view(1, split.P, C)
