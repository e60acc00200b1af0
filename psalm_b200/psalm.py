"""`PSALM` — the drop-in object for the reference's segmentation inference path.

Keeps the operator surface of `PSALM(PhiForCausalLM, LlavaMetaForCausalLM)` that the eval scripts use
(reference language_model/llava_phi.py:146, psalm/model/llava_arch.py:49-63):
    model.eval_seg(input_ids=..., attention_mask=..., images=..., seg_info=..., class_name_ids=...,
                   cls_indices=..., class_name_embedding_indices=..., token_refer_id=...,
                   refer_embedding_indices=..., is_thing_list=...)      -> list[dict]   (llava_phi.py:1317)
    model.get_model(), model.get_vision_tower(), model.encode_images(images),
    model.get_vision_tower_feature(images), model.pixel_decoder.forward_features(dict),
    model.predictor(x, mask_features, None, seg_query, SEG_embedding, class_name_embedding, None)
and loads the reference checkpoint layout unchanged (layout.py / loader.py).

With `use_cuda_graph=True` the network and the device part of the task heads replay from one CUDA graph;
the returned tensors then alias the graph's static buffers and are valid until the next `eval_seg` call on
the same model (consume or clone them first, as the reference's eval loops do with `evaluator.process`).

How it differs from the reference on purpose (results are unchanged, see DESIGN.md):
  * Swin runs ONCE per image (the reference runs it twice on identical input, llava_phi.py:449 and :223);
  * every image of the batch is post-processed (the reference returns inside the loop, llava_phi.py:1472);
  * no CPU / PyTorch fallback for the hot operators: a missing CUDA library raises.
"""
import contextlib
import copy
from collections import OrderedDict

import torch
import torch.nn.functional as F

from . import postprocess as PP
from . import sequence as SEQ
from .layout import PsalmConfig
from .mask_decoder import MultiScaleMaskedTransformerDecoderForOPTPreTrain
from .phi import PhiModel
from .pixel_decoder import MSDeformAttnPixelDecoder
from .projector import ResNetSwin
from .swin import SwinTransformer


class StagedImages:
    """A batch of images whose host->device copy was enqueued on the model's copy stream by
    `PSALM.stage_images`; `PSALM.eval_seg(images=staged, ...)` waits for it on the compute stream."""

    def __init__(self, slot, ready):
        self.slot, self.ready = slot, ready          # slot = [device buffer, event "consumer is done"]
        self.tensor = slot[0]
        self.shape, self.dtype = slot[0].shape, slot[0].dtype


class PendingSeg:
    """Handle of a submitted `PSALM.eval_seg_async` or `ImageSession.eval_seg_async` call: the device work is queued
    (graph replays), and when the graph holds the device part of the task heads, the few integers the host merge needs
    are on their way to pinned memory.  `result()` finishes the post-processing ON THE CALLER'S CURRENT STREAM (after
    making it wait for the pass), so a caller that wants the host work of image batch k to overlap the device work of
    batch k+1 submits k+1 first and calls `result()` of k under a side stream.  The tensors of the result live in the
    lane's static buffers: they stay valid until the next submission on the same lane.

    `parts`: one (out, hostvecs, is_thing_list) per forward output (one for an image batch, one per prompt of a
    session), post-processed with the `thresholds` (object mask, overlap) of the submission."""

    def __init__(self, model, parts, image_hw, seg_info, boxes, done, thresholds, mask_format="dense"):
        self.model, self.parts, self.image_hw, self.seg_info, self.boxes = model, parts, image_hw, seg_info, boxes
        self.done, self.thresholds, self.mask_format = done, thresholds, mask_format

    def result(self):
        m = self.model
        if self.done is not None:
            torch.cuda.current_stream(m.device).wait_event(self.done)
        if any(hostvecs is not None for _, hostvecs, _ in self.parts):
            self.done.synchronize()                          # pinned host vectors are complete
        results = None
        for out, hostvecs, things in self.parts:
            res = m.post_process(out, self.image_hw, self.seg_info, self.boxes, hostvecs, things, *self.thresholds)
            results = res if results is None else results + res
        if self.mask_format == "rle":
            attach_rle(results)
        return results


class ImageSession:
    """One image opened by `PSALM.open_image`: its Swin maps, projector tokens, pixel-decoder outputs and decoder K / V
    projections are computed once, and the prompt-independent prefix of every prompt set is prefilled once (its K / V
    of all layers kept for the two most recent prefixes).  `eval_seg(prompts)` then runs only the prompt suffixes.
    Valid until the next `open_image` on the same lane (a stale session raises RuntimeError)."""

    MAX_PREFIXES = 2

    def __init__(self, model, lane, gen, state, image_hw, seg_info, boxes):
        self.model, self.lane, self.gen, self.state = model, lane, gen, state
        self.image_hw, self.seg_info, self.boxes = image_hw, seg_info, boxes
        self.prefixes = OrderedDict()     # prefix input ids (bytes) -> PagedKVCache of its K / V

    def _region_inputs(self, regions):
        """The regions of all prompts of a call, rasterised in one batch at the session's geometry (original size, un-padded
        box, input size) -> (bits, row_prefix, sample-point indices [R,256] on the device).  The set-pixel counts come to
        the host (the reference draws its points there), and the indices are drawn region by region in prompt order: the
        draws of per-prompt eval_seg calls made in that order from the same generator."""
        from .region import draw_point_indices, rasterize_visual_prompts
        m = self.model
        info = self.seg_info[0]
        H, W = self.image_hw
        bits, prefix, count = rasterize_visual_prompts(regions, info.get("height", H), info.get("width", W),
                                                       tuple(self.boxes[0]), (H, W), m.device)
        sel = draw_point_indices(count.tolist())
        return bits, prefix, sel.to(m.device)

    def prefix_cache(self, split):
        """K / V of the shared prefix `split` (prefilled on first use, two most recent prefixes kept)."""
        key = split.prefix_ids.tobytes()
        cache = self.prefixes.get(key)
        if cache is None:
            m = self.model
            cache = m._phase("_prefix_graphs", (self.lane, key), lambda sp: m._prefix_core(self.state, sp),
                             refresh=(split,), reads=(self.state,))
            while len(self.prefixes) >= self.MAX_PREFIXES:
                self.prefixes.popitem(last=False)
            self.prefixes[key] = cache
        self.prefixes.move_to_end(key)
        return cache

    @torch.no_grad()
    def eval_seg(self, prompts, is_thing_list=None, mask_format="dense"):
        """results[k] == model.eval_seg(images, seg_info, **prompts[k])[0] (same structure; values within the tolerances
        of a split prefill).  A prompt dict may carry its own `is_thing_list` (panoptic prompts with different class
        lists); it overrides the call-level one.

        Interactive segmentation (the "region" task): a prompt with K <region> tokens carries `visual_prompts`, K
        (kind, source) pairs at the original image size - kind "point", "scribble", "box" or "mask"; source a COCO RLE
        dict, a binary [height, width] tensor, a (row, col) click or a (min_row, min_col, max_row, max_col) box
        (region.rasterize_visual_prompts).  The regions are rasterised on the device as the reference mapper prepares
        them (coco_instance_mapper.py:233-251) and their sample points are drawn like eval_seg's, prompt by prompt, from
        the global CPU generator; the result is eval_seg's for the region task (instances with pred_masks [Q,H,W] and
        scores [Q,K]; `gt` when the opened image's seg_info carries instances.gt_masks)."""
        return self.eval_seg_async(prompts, is_thing_list, mask_format).result()

    @torch.no_grad()
    def eval_seg_async(self, prompts, is_thing_list=None, mask_format="dense"):
        if mask_format not in MASK_FORMATS:
            raise ValueError("mask_format must be one of %s, got %r" % (MASK_FORMATS, mask_format))
        m = self.model
        m._check_lane(self.lane, self.gen, "stale ImageSession: open_image was called again on lane %d")
        things = [p.get("is_thing_list", is_thing_list) for p in prompts]
        if m.panoptic_on and any(t is None for t in things):
            raise ValueError("is_thing_list need to be given")   # llava_phi.py:1337-1339
        visual = any("visual_prompts" in p for p in prompts)
        if visual and not m.region_on:
            raise ValueError("visual_prompts need the model in the \"region\" task (got %r)" % m.seg_task)
        split, plan = m._cached_split(prompts, self.image_hw)
        region = None
        if visual and plan.region_counts is not None:
            vps = [p.get("visual_prompts", ()) for p in prompts]
            if tuple(len(v) for v in vps) != plan.region_counts:
                raise ValueError("visual_prompts: %s regions for %s <region> tokens" % (
                    tuple(len(v) for v in vps), plan.region_counts))
            m._region_projector()
            m._region_side(split.img_pos.numel())
            region = self._region_inputs([r for v in vps for r in v])
        outs = m._prompts_forward(self, split, plan, region)
        done = None
        if m.device.type == "cuda":
            done = torch.cuda.Event()
            done.record(torch.cuda.current_stream(m.device))
        return PendingSeg(m, [(out, None, t) for out, t in zip(outs, things)], self.image_hw, self.seg_info[:1],
                          self.boxes[:1], done, (m.object_mask_threshold, m.overlap_threshold), mask_format)


MASK_FORMATS = ("dense", "rle")


def _content_key(t):
    """Hashable key of a prompt tensor (or a list of them) by content: the plan caches are keyed by what the prompt says."""
    if t is None:
        return None
    if isinstance(t, (list, tuple)):
        return tuple(_content_key(x) for x in t)
    t = torch.as_tensor(t).detach().cpu().contiguous()
    return (tuple(t.shape), str(t.dtype), t.numpy().tobytes())


# The device tensors a CUDA graph reads from a plan input of a phase (PSALM._phase), by plan type
_GRAPH_TENSORS = {SEQ.SequencePlan: ("tok_ids", "img_pos", "seg_pos", "pad_pos", "attention_mask", "cls_pool", "refer_pool",
                                      "region_pos"),
                  SEQ.PromptSplit: ("tok_ids", "img_pos")}


def _plan_key(plan):
    """The structure of a SequencePlan a captured graph is bound to (shapes, which optional rows exist, and the regions
    per row of a plan with <region> rows)."""
    key = (plan.B, plan.T, plan.n_img, plan.any_padding, None if plan.cls_pool is None else tuple(plan.cls_pool.shape),
           plan.refer_pool is not None, None if plan.pad_pos is None else int(plan.pad_pos.numel()))
    return key if plan.region_counts is None else key + (tuple(plan.region_counts),)


def attach_rle(results):
    """mask_format="rle": `instances.pred_masks_rle` = pycocotools RLE dicts of `instances.pred_masks` (same order) for
    every result with instances.  The masks of all images of a size are encoded in one batch on the device."""
    from . import rle
    groups = {}
    for r in results:
        inst = r.get("instances")
        if inst is not None:
            m = inst.pred_masks
            groups.setdefault((tuple(m.shape[1:]), m.dtype, m.device), []).append(inst)
    for insts in groups.values():
        dicts = rle.to_dicts(rle.encode_device([i.pred_masks for i in insts]))
        pos = 0
        for inst in insts:
            k = inst.pred_masks.shape[0]
            inst.pred_masks_rle = dicts[pos:pos + k]
            pos += k


class PSALMModel:
    """`model.model` of the reference (PSALMModel(LlavaMetaModel, PhiModel), llava_phi.py:52): owns the
    LLM, the vision tower and the projector."""

    def __init__(self, sd, cfg, dtype, device):
        self.phi = PhiModel(sd, "model.", cfg.phi, dtype, device)
        self.embed_tokens = self.phi.embed_tokens
        self.vision_tower = SwinTransformer(sd, "model.vision_tower.", cfg.swin, dtype, device)
        self.mm_projector = ResNetSwin(sd, "model.mm_projector.", dtype, device)

    def get_vision_tower(self):
        return self.vision_tower

    def __call__(self, inputs_embeds=None, attention_mask=None, **_):
        return self.phi(inputs_embeds, attention_mask)


class PSALM:
    def __init__(self, state_dict, cfg: PsalmConfig = PsalmConfig(), dtype=torch.bfloat16, device="cuda",
                 seg_task="panoptic", use_cuda_graph=False):
        self._check_runtime(device)
        self.use_cuda_graph = use_cuda_graph
        self._lane_gen = {}            # lane -> generation of its newest session (open_image / open_video)
        # one fused kernel for the task heads (16-bit storage); fp32 parity runs keep the exact torch path
        self._fused_postprocess = dtype != torch.float32
        self.overlap_branches = True   # pixel decoder || LLM prefill on two streams
        self.cfg, self.dtype, self.device = cfg, dtype, torch.device(device)
        sd = state_dict
        cv = lambda t: t.to(device=device, dtype=dtype).contiguous()  # noqa: E731
        self.model = PSALMModel(sd, cfg, dtype, device)
        self.pixel_decoder = MSDeformAttnPixelDecoder(sd, "pixel_decoder.", cfg.mask, dtype, device)
        self.predictor = MultiScaleMaskedTransformerDecoderForOPTPreTrain(sd, "predictor.", cfg.mask, dtype, device)
        self.seg_query = cv(sd["seg_query"])
        self.proj = {n: (cv(sd[n + ".weight"]), cv(sd[n + ".bias"]))
                     for n in ("seg_query_projector", "SEG_token_projector", "class_name_projector", "region_projector")
                     if n + ".weight" in sd}     # region_projector is optional in the checkpoint contract (loader.py)
        # lm_head (no bias in the reference, llava_phi.py:191): only the chat / decode path reads it
        self.lm_head = None
        if "lm_head.weight" in sd:
            self.lm_head = (cv(sd["lm_head.weight"]), cv(sd["lm_head.bias"]) if "lm_head.bias" in sd else None)
        self.num_queries = cfg.mask.num_queries
        self.test_topk_per_image = cfg.mask.num_queries
        self.size_divisibility = cfg.mask.size_divisibility
        # panoptic thresholds: the reference hard-codes 0.8 / 0.8 (llava_phi.py:331-332)
        self.object_mask_threshold = cfg.mask.object_mask_threshold
        self.overlap_threshold = cfg.mask.overlap_threshold
        self.set_task(seg_task)

    @contextlib.contextmanager
    def _precision_scope(self):
        """fp32 models run true fp32 library GEMMs / convolutions (cuDNN and cuBLAS would otherwise pick TF32);
        the global switches are restored on exit, other models in the process are not affected."""
        if self.dtype != torch.float32:
            yield
            return
        old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        try:
            yield
        finally:
            torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old

    @staticmethod
    def _check_runtime(device):
        """No CPU path and no silent fallback: refuse to construct without a GPU and the built kernels."""
        if torch.device(device).type != "cuda" or not torch.cuda.is_available():
            raise RuntimeError("psalm_b200.PSALM needs a CUDA device: there is no CPU implementation of the hot path")
        from . import _lib
        _lib.lib()

    @property
    def fused_postprocess(self):
        """Fused task-head kernels: 16-bit storage, and not the region task (its head is a [K,Q] score table over the
        plain thresholded masks, done with torch ops)."""
        return self._fused_postprocess and not getattr(self, "region_on", False)

    @fused_postprocess.setter
    def fused_postprocess(self, v):
        self._fused_postprocess = bool(v)

    # ---- configuration (llava_phi.py:268-301) ----------------------------------------------------
    def set_task(self, seg_task):
        if seg_task not in ("semantic", "instance", "panoptic", "referring", "region"):
            raise NotImplementedError("SEG_TASK %r (the video variant is outside this build's scope)" % seg_task)
        self.seg_task = seg_task
        self.semantic_on = seg_task in ("semantic", "panoptic")
        self.instance_on = seg_task in ("instance", "panoptic")
        self.panoptic_on = seg_task == "panoptic"
        self.referring_on = seg_task == "referring"
        self.region_on = seg_task == "region"
        self.sem_seg_postprocess_before_inference = self.instance_on or self.panoptic_on or self.referring_on or self.region_on

    @classmethod
    def from_state_dict(cls, sd, **kw):
        return cls(sd, **kw)

    @classmethod
    def from_pretrained(cls, model_path, mask_decoder_cfg=None, **kw):
        """Checkpoint directory of the reference (config.json + safetensors / bin shards), keys unchanged
        (psalm/model/builder.py:55 calls this on the reference class)."""
        from .builder import from_pretrained
        return from_pretrained(cls, model_path, mask_decoder_cfg, **kw)

    def generate(self, input_ids=None, images=None, max_new_tokens=32, do_sample=False, temperature=1.0, top_p=None,
                 eos_token_id=None, **_unused):
        """Chat / decoding path (psalm/serve/cli.py:89-96): prefill + autoregressive decode with a paged KV cache
        (psalm_b200/generate.py).  Returns the NEW token ids [B, n_new]."""
        from .generate import generate
        return generate(self, input_ids, images, max_new_tokens, do_sample, temperature, top_p, eos_token_id)

    # ---- LlavaMetaForCausalLM methods the training / serving scripts call by name -------------------
    def initialize_vision_tokenizer(self, model_args, tokenizer):
        """llava_arch.py:181-217.  The released checkpoints set mm_use_im_patch_token = mm_use_im_start_end = False, for
        which the reference method does nothing; growing the embedding table is a training-time operation."""
        if getattr(model_args, "mm_use_im_patch_token", False) or getattr(model_args, "mm_use_im_start_end", False):
            raise NotImplementedError("adding image patch / start / end tokens resizes the embedding table: training-time "
                                      "surface, outside this inference build")

    def prepare_inputs_labels_for_multimodal(self, input_ids, attention_mask, past_key_values, labels, images,
                                             class_name_embedding_indices=None, class_name_ids=None, cls_indices=None,
                                             instances=None, token_refer_id=None, refer_embedding_indices=None):
        """llava_phi.py:767-971: sentinel ids -> embeddings.  Returns the reference's tuple
        (input_ids=None, attention_mask, past_key_values, inputs_embeds, labels, seg_query_mask,
         class_name_embedding_indices, region_embedding_masks, refer_embedding_indices) for the image-prefill case."""
        with self._precision_scope():
            img_tok = self.encode_images(images.to(self.device))
        plan = self.make_plan(input_ids, attention_mask, images.shape[-2:], class_name_ids, cls_indices,
                              class_name_embedding_indices, token_refer_id, refer_embedding_indices)
        region_mask = None
        region_feat = None
        if plan.region_pos is not None:    # llava_phi.py:791-797: region features from the instances' region masks
            if instances is None:
                raise ValueError("<region> tokens in the prompt need `instances` with region_masks (llava_phi.py:791-792)")
            from .region import region_inputs
            plan.region_points, plan.region_image, counts = region_inputs([dict(instances=i) for i in instances])
            assert counts == plan.region_counts, "the munber of <region> tokens and regions needs to be same"
        plan = plan.to(self.device)
        if plan.region_pos is not None:
            region_feat = self._region_features(img_tok, plan)
        embeds = SEQ.materialize_embeds(plan, self.model.embed_tokens, img_tok, self.seg_query, region_feat)
        B, T = plan.B, plan.T
        flat = lambda pos: torch.zeros(B * T, device=self.device).index_fill_(0, pos, 1.0).view(B, T)   # noqa: E731
        seg_query_mask = flat(plan.seg_pos)
        cls_idx = None
        if plan.cls_pool is not None:     # class index (1-based) of every position, 0 elsewhere (:671-673)
            cls_idx = ((plan.cls_pool > 0).float() * torch.arange(1, plan.cls_pool.shape[1] + 1, device=self.device)
                       .view(1, -1, 1)).sum(1).long()
        ref_idx = (plan.refer_pool[:, 0] > 0).long() if plan.refer_pool is not None else None
        if plan.region_pos is not None:
            region_mask = flat(plan.region_pos)
        return None, plan.attention_mask, past_key_values, embeds, labels, seg_query_mask, cls_idx, region_mask, ref_idx

    def _region_features(self, img_tok, plan):
        """[R, hidden] pooled region features (region_pooling, context_cluster.py:333-400) from the projector tokens."""
        from . import kernels
        side = self._region_side(img_tok.shape[1])
        return kernels.region_pool(img_tok.contiguous(), plan.region_points, plan.region_image, side, side)

    @staticmethod
    def _region_side(n_img):
        """Side of the projector map that region pooling reads: context_cluster.py:355 takes h = w = int(sqrt(n)), so
        square maps only."""
        side = int(round(n_img ** 0.5))
        if side * side != n_img:
            raise ValueError("region prompts need a square projector map (got %d tokens)" % n_img)
        return side

    def _region_projector(self):
        if "region_projector" not in self.proj:
            raise KeyError("region prompts need region_projector.* in the checkpoint")
        return self.proj["region_projector"]

    # ---- LlavaMetaForCausalLM surface --------------------------------------------------------------
    def get_model(self):
        return self.model

    def get_vision_tower(self):
        return self.model.get_vision_tower()

    def encode_images(self, images):
        """llava_phi.py:448-451."""
        with self._precision_scope():
            feats = self.get_vision_tower()(images)
            return self.model.mm_projector(feats[-1])

    def get_vision_tower_feature(self, images):
        """llava_phi.py:222-230."""
        with self._precision_scope():
            f = self.get_vision_tower()(images)
        return dict(res2=f[0], res3=f[1], res4=f[2], res5=f[3])

    # ---- the hot path -----------------------------------------------------------------------------
    @torch.no_grad()
    def forward_core(self, images, plan, trace=None):
        """Device-only part of eval_seg: images [B,3,H,W] on device, `plan` a SequencePlan on device.
        Returns dict(pred_masks [B,Q,H4*W4], mask_size, pred_class_name_logits, pred_SEG_logits).
        `trace`: optional dict that receives the stage outputs (token-major), for the per-stage parity tests."""
        with self._precision_scope():
            return self._forward_core(images, plan, trace)

    def _swin_project(self, images):
        """Swin (once) and the projector: (Swin token maps, their sizes, projector tokens [B,n_img,hidden])."""
        toks, sizes = self.model.vision_tower.forward_tokens(images)
        h5, w5 = sizes[3]
        img_tok = self.model.mm_projector(toks[3].view(toks[3].shape[0], h5, w5, -1).permute(0, 3, 1, 2))
        return toks, sizes, img_tok

    def _llm_heads(self, plan, hidden):
        """(seg queries, SEG embedding, class-name embeddings, projected <region> rows) from the LLM's hidden states; None
        for a head the prompt has no rows for."""
        seg_q = F.linear(SEQ.gather_seg_query(plan, hidden), *self.proj["seg_query_projector"])
        SEG_emb = cls_emb = region_rows = None
        if plan.refer_pool is not None:
            SEG_emb = F.linear(SEQ.pool(plan.refer_pool, hidden), *self.proj["SEG_token_projector"])
        if plan.cls_pool is not None:
            cls_emb = F.linear(SEQ.pool(plan.cls_pool, hidden), *self.proj["class_name_projector"])
        if plan.region_pos is not None:     # llava_phi.py:1385-1388: hidden states at the <region> rows -> region_projector
            region_rows = F.linear(SEQ.gather_region_rows(plan, hidden), *self._region_projector())
        return seg_q, SEG_emb, cls_emb, region_rows

    def _forward_core(self, images, plan, trace=None):
        toks, sizes, img_tok = self._swin_project(images)
        # The pixel decoder needs only the Swin maps, the LLM only the projector tokens: the two branches run on two
        # streams (also inside a captured graph) and meet at the mask decoder.  The LLM branch is a chain of library GEMMs
        # at the tensor-core peak whose last waves leave SMs idle; the pixel decoder's memory-bound kernels fill them.
        branch, main = None, None
        if self.overlap_branches and toks[0].is_cuda and torch.cuda.is_current_stream_capturing():
            # (graph capture only: eager launches are host bound, two streams would buy nothing there)
            main = torch.cuda.current_stream(self.device)
            if not hasattr(self, "_branch_stream"):
                self._branch_stream = torch.cuda.Stream(device=self.device)
            self._branch_stream.wait_stream(main)
            with torch.cuda.stream(self._branch_stream):
                branch = self.pixel_decoder.forward_tokens(toks, sizes)
            for t in toks:
                t.record_stream(self._branch_stream)
        region_feat = None
        if plan.region_pos is not None:
            src_tok = img_tok
            if plan.vp_images is not None:   # DAVIS variant: pooled from the visual-prompt frame's map (llava_phi.py:1665-1670)
                src_tok = self._swin_project(plan.vp_images)[2]
            region_feat = self._region_features(src_tok, plan)
        embeds = SEQ.materialize_embeds(plan, self.model.embed_tokens, img_tok, self.seg_query, region_feat)
        # (cutting the batch into groups on separate streams so that the prefill GEMMs fill each other's tail waves was
        # measured and is slower: 20.8 ms / 21.9 ms per step of 4 for 2 / 4 groups against 19.5 ms)
        hidden = self.model.phi(embeds, plan.attention_mask if plan.any_padding else None)
        seg_q, SEG_emb, cls_emb, rows = self._llm_heads(plan, hidden)
        region_emb = None if rows is None else list(torch.split(rows, list(plan.region_counts), 0))
        if branch is None:
            mask_features, ms, ms_sizes = self.pixel_decoder.forward_tokens(toks, sizes)
        else:   # join the pixel-decoder branch
            mask_features, ms, ms_sizes = branch
            main.wait_stream(self._branch_stream)
            for t in [mask_features] + list(ms):
                t.record_stream(main)
        out = self.predictor.forward_tokens(ms, ms_sizes, mask_features, sizes[0], seg_q, SEG_emb, cls_emb,
                                            region_embedding_list=region_emb)
        out["mask_size"] = sizes[0]
        if trace is not None:
            trace.update(region_features=region_feat, region_emb=region_emb)
            trace.update(swin=toks, swin_sizes=sizes, img_tok=img_tok, embeds=embeds, hidden=hidden, seg_query=seg_q,
                         SEG_emb=SEG_emb, cls_emb=cls_emb, mask_features=mask_features, ms=ms, ms_sizes=ms_sizes)
        return out

    # ---- CUDA-graph replay of the device-only part -------------------------------------------------
    # Every graph table is a bounded LRU: each entry owns static buffers + a private pool (hundreds of MB at 1024^2, B = 4)
    MAX_GRAPHS = 8
    MAX_PLANS = 16

    def _lru(self, table, key, make, bound):
        """The entry of `key` in the bounded LRU cache `self.<table>`, made by `make()` on a miss; when the table is
        full the least recently used entry goes."""
        cache = self.__dict__.setdefault(table, OrderedDict())
        ent = cache.get(key)
        if ent is None:
            ent = make()
            while len(cache) >= bound:
                cache.popitem(last=False)
            cache[key] = ent
        cache.move_to_end(key)
        return ent

    def _capture(self, fn):
        """(CUDA graph of fn(), its output): two warm-up calls on a side stream, then the capture."""
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(side), self._precision_scope():
            for _ in range(2):
                fn()
        torch.cuda.current_stream(self.device).wait_stream(side)
        torch.cuda.synchronize(self.device)
        g = torch.cuda.CUDAGraph()
        with self._precision_scope(), torch.cuda.graph(g):
            out = fn()
        return g, out

    def _phase(self, table, key, fn, refresh=(), reads=()):
        """fn(*refresh), launched eagerly under `_precision_scope`, or with `use_cuda_graph` replayed from the CUDA graph of
        `key` in the bounded LRU `self.<table>`; a graph's output is its static buffers, overwritten by its next replay.
        `refresh`: the inputs that change per call (tensors, SequencePlans, PromptSplits); a graph reads its own copies of
        their device tensors (`_GRAPH_TENSORS`), refreshed before every replay, since a cached input may be evicted and
        freed while the graph lives.  `reads`: objects whose buffers fn reads as they are; their identities complete the
        key and the entry holds them, so that an id cannot be handed to a new object while the graph lives."""
        if not self.use_cuda_graph:
            with self._precision_scope():
                return fn(*refresh)

        def tensors(x):
            return [x] if isinstance(x, torch.Tensor) else [getattr(x, n) for n in _GRAPH_TENSORS[type(x)]]

        def static_copy(x):
            if isinstance(x, torch.Tensor):
                return x.clone()
            static = copy.copy(x)
            for n in _GRAPH_TENSORS[type(x)]:
                t = getattr(x, n)
                setattr(static, n, None if t is None else t.clone())
            return static

        def make():
            static = [static_copy(x) for x in refresh]
            g, out = self._capture(lambda: fn(*static))
            return g, static, out, reads
        g, static, out, _ = self._lru(table, key + tuple(id(r) for r in reads), make, self.MAX_GRAPHS)
        for s, x in zip(static, refresh):
            for dst, src in zip(tensors(s), tensors(x)):
                if src is not None:
                    dst.copy_(src, non_blocking=True)
        g.replay()
        return out

    def _forward_post(self, images, plan, geoms):
        """forward_core, plus the device part of the fused task heads for the per-image geometries `geoms` when every
        image takes the fused kernel (capturable)."""
        out = self._forward_core(images, plan)
        if geoms is not None:
            hw = tuple(images.shape[-2:])
            routes = self._routes(hw, geoms, out)
            if all(r is not None for r in routes):
                out["post"] = self._post_device(out, hw, routes, getattr(self, "is_thing_list", None),
                                                self.object_mask_threshold)
                out["post_geoms"] = geoms
        return out

    @torch.no_grad()
    def forward_core_graphed(self, images, plan, lane=0, fuse_post=True):
        """Same results as forward_core, replayed from a CUDA graph captured per (image size, prompt
        structure): the ~800 launches of one image become one graph launch (the reference issues them
        one by one from Python, plus ~150 extra tiny launches in its decoder).  `lane` selects an
        independent graph + static buffers so that several images can be in flight on different streams.
        `fuse_post` (`_fused_applies`): True (no crop / resize) or a tuple of per-image geometries puts the device part
        of the fused task heads into the graph; False leaves the task heads to `post_process`.  Without `use_cuda_graph`
        the same work is launched eagerly."""
        key = (lane, fuse_post, self.seg_task, float(self.object_mask_threshold),
               tuple(getattr(self, "is_thing_list", None) or ()), tuple(images.shape), str(images.dtype)) + _plan_key(plan)
        geoms = None
        if isinstance(fuse_post, tuple):
            geoms = fuse_post
        elif fuse_post:
            Hp, Wp = self._padded(images.shape[-2:])
            geoms = ((Hp, Wp, Hp, Wp),) * images.shape[0]      # no crop / resize
        return self._phase("_graphs", key, lambda img, p: self._forward_post(img, p, geoms), refresh=(images, plan))

    # ---- sessions: several prompts against one image, the frames of a clip ------------------------------------------
    def _open_lane(self, lane):
        """Generation of a new session on `lane`.  The phases of a lane share static buffers, so the new session ends the
        lane's earlier ones."""
        self._lane_gen[lane] = self._lane_gen.get(lane, 0) + 1
        return self._lane_gen[lane]

    def _check_lane(self, lane, gen, stale):
        """RuntimeError(`stale` % lane) when the session of generation `gen` on `lane` has been ended."""
        if self._lane_gen.get(lane) != gen:
            raise RuntimeError(stale % lane)

    @torch.no_grad()
    def open_image(self, images, seg_info, lane=0):
        """Encode ONE image (images [1,3,H,W]: float, uint8 or StagedImages, as eval_seg) for several prompts: Swin, the
        projector, the pixel decoder and the decoder's K / V projections run once; returns an `ImageSession` whose
        `eval_seg(prompts)` runs only what depends on the prompts.  Opening an image ends the previous session of `lane`."""
        if images.shape[0] != 1 or len(seg_info) != 1:
            raise ValueError("open_image takes one image (got %d)" % images.shape[0])
        gen = self._open_lane(lane)
        state = self._encode_image(self._device_images(images), lane)
        self._release_staged(images)
        _, boxes = self._fused_applies(images.shape[-2:], seg_info)
        return ImageSession(self, lane, gen, state, tuple(images.shape[-2:]), list(seg_info), boxes)

    # The session phases, graphed per lane: the image (per image shape and dtype), the prefix prefill (per image state and
    # prefix content), the prompt pass (per image state, prefix cache, plan structure and task) and the video prompt
    # phase (per image state and clip buffers).  Later phases read the static buffers of the earlier ones of the same
    # lane, so a session is valid until the next open_image / open_video on its lane.
    def _encode_image(self, images, lane):
        return self._phase("_image_graphs", (lane, tuple(images.shape), str(images.dtype)), self._image_core,
                           refresh=(images,))

    def _image_core(self, images):
        """Prompt-independent device work of one image (capturable)."""
        toks, sizes, img_tok = self._swin_project(images)
        mask_features, ms, ms_sizes = self.pixel_decoder.forward_tokens(toks, sizes)
        mem = self.predictor.memory(ms, ms_sizes, mask_features, sizes[0], self.num_queries)
        return dict(swin=toks, swin_sizes=sizes, img_tok=img_tok, mask_features=mask_features, ms=ms, ms_sizes=ms_sizes,
                    mem=mem, mask_size=sizes[0])

    def _prefix_core(self, state, split):
        """Prefill of the shared prefix (split.tok_ids / img_pos on the device) into a new PagedKVCache of one page that
        holds the P rows rounded up to 64 (head-major [nh, P_pad, hd] per layer, the layout psalm_prefix_causal_attention
        reads); capturable.  The rows are written from row 0 (the cache's seq_lens stay 0, so a replay writes the same
        rows again); the host-side length P is what forward_suffix reads."""
        from .generate import PagedKVCache
        page = -(-split.P // 64) * 64
        cache = PagedKVCache(self.cfg.phi, 1, page, self.dtype, self.device, page_size=page)
        self.model.phi.forward(SEQ.prefix_embeds(split, self.model.embed_tokens, state["img_tok"]), None, cache=cache)
        cache.length = split.P
        return cache

    def _prompts_core(self, state, cache, plan, region=None, image_hw=None):
        """Device work of K prompt suffixes (plan on device) against an opened image and its prefix cache (capturable).
        Returns forward_core's dict for the K prompts (pred_masks [K,Q,H4*W4], ...) and the suffix hidden states.
        `region`: (bits, row_prefix, sample-point indices) of the R regions of the prompts (ImageSession._region_inputs),
        pooled from the image's projector tokens; `image_hw` is the size the bits are at."""
        from . import kernels
        img_tok = state["img_tok"]
        region_feat = None
        if region is not None:
            bits, prefix, sel = region
            R, dev = sel.shape[0], sel.device
            side = self._region_side(img_tok.shape[1])
            pts = kernels.region_points_gather(bits, prefix, sel, torch.arange(R, dtype=torch.int32, device=dev), *image_hw)
            region_feat = kernels.region_pool(img_tok.contiguous(), pts, torch.zeros(R, dtype=torch.int32, device=dev),
                                              side, side)
        embeds = SEQ.materialize_embeds(plan, self.model.embed_tokens, img_tok[:, :0], self.seg_query, region_feat)
        hidden = self.model.phi.forward_suffix(embeds, cache, plan.attention_mask if plan.any_padding else None)
        seg_q, SEG_emb, cls_emb, rows = self._llm_heads(plan, hidden)
        region_emb = None if rows is None else list(torch.split(rows, list(plan.region_counts), 0))
        out = self.predictor.forward_tokens(None, state["ms_sizes"], None, state["mask_size"], seg_q, SEG_emb, cls_emb,
                                            region_embedding_list=region_emb, memory=state["mem"])
        out["mask_size"] = state["mask_size"]
        out["hidden"], out["seg_query"] = hidden, seg_q
        return out

    def _cached_split(self, prompts, image_hw):
        """(host PromptSplit, device suffix plan) of a prompt set, cached by content like `_cached_plan`."""
        key = (tuple(image_hw),) + tuple(tuple(_content_key(p.get(n)) for n in SEQ.PROMPT_KEYS) + ("visual_prompts" in p,)
                                         for p in prompts)

        def make():
            import dataclasses
            split = SEQ.split_prompts(prompts, self.make_plan_n_img(image_hw), self.num_queries)
            plan = split.suffix.to(self.device)
            split = dataclasses.replace(split, tok_ids=split.tok_ids.to(self.device), img_pos=split.img_pos.to(self.device),
                                        suffix=None)
            return split, plan
        return self._lru("_splits", key, make, self.MAX_PLANS)

    def make_plan_n_img(self, image_hw):
        """Projector tokens of an image of size image_hw (the <image> expansion of make_plan)."""
        H, W = image_hw
        ps = self.cfg.swin.patch
        h, w = -(-H // ps), -(-W // ps)
        for _ in range(len(self.cfg.swin.depths) - 1):
            h, w = (h + 1) // 2, (w + 1) // 2
        return ((h - 1) // 2 + 1) * ((w - 1) // 2 + 1)   # conv3x3 stride 2 pad 1 of the projector

    def _prompts_forward(self, sess, split, plan, region=None):
        """Run the prompt pass of a session and cut its output into one forward_core-style dict per prompt.  `region`: the
        device inputs of the prompts' regions (ImageSession._region_inputs); the graph reads its own copies of them."""
        cache = sess.prefix_cache(split)
        out = self._phase("_prompt_graphs", (sess.lane, self.seg_task) + _plan_key(plan),
                          lambda p, *reg: self._prompts_core(sess.state, cache, p, reg or None, sess.image_hw),
                          refresh=(plan,) + tuple(region or ()), reads=(sess.state, cache))
        outs = []
        for k, ncls in enumerate(split.n_classes):
            cls = out["pred_class_name_logits"]
            seg = out["pred_SEG_logits"]
            reg = out["pred_region_logits"]
            outs.append(dict(pred_masks=out["pred_masks"][k:k + 1], mask_size=out["mask_size"],
                             pred_class_name_logits=None if cls is None else cls[k:k + 1, :, :ncls].contiguous(),
                             pred_SEG_logits=None if seg is None else seg[k:k + 1],
                             pred_region_logits=None if reg is None else [reg[k]]))
        return outs

    # ---- input staging: overlap the upload of batch k+1 with the compute of batch k ----------------------
    def stage_images(self, images_host):
        """Enqueue the host->device copy of a (pinned) image batch on a dedicated copy stream and return a
        `StagedImages` handle for `eval_seg`.  Two device buffers per (shape, dtype) alternate; a buffer is reused
        only after the pass that consumed it has read it (event recorded by eval_seg)."""
        if not hasattr(self, "_stage"):
            self._stage = dict(stream=torch.cuda.Stream(device=self.device), rings={}, count={})
        st = self._stage
        key = (tuple(images_host.shape), images_host.dtype)
        ring = st["rings"].setdefault(key, [[torch.empty(images_host.shape, dtype=images_host.dtype, device=self.device),
                                             None] for _ in range(2)])
        n = st["count"].get(key, 0)
        st["count"][key] = n + 1
        slot = ring[n % 2]
        with torch.cuda.stream(st["stream"]):
            if slot[1] is not None:
                st["stream"].wait_event(slot[1])
            slot[0].copy_(images_host, non_blocking=True)
            ready = torch.cuda.Event()
            ready.record(st["stream"])
        return StagedImages(slot, ready)

    def _device_images(self, images):
        """`images` (a tensor or StagedImages) as a device tensor.  Float images are the reference contract (already
        normalised by the mapper); uint8 images are raw pixel values, normalised on the device (coco_panoptic_mapper.py:161)
        - 4x fewer bytes over PCIe.  A StagedImages upload is already in flight on the copy stream: the current stream
        waits for it, and `_release_staged` must follow the pass that reads it."""
        if isinstance(images, StagedImages):
            torch.cuda.current_stream(self.device).wait_event(images.ready)
            return images.tensor
        return images.to(self.device, non_blocking=True)

    def _release_staged(self, images):
        """After the pass that reads `images` is enqueued: a staging buffer may be overwritten once that pass has run."""
        if isinstance(images, StagedImages):
            images.slot[1] = torch.cuda.Event()
            images.slot[1].record(torch.cuda.current_stream(self.device))

    def make_plan(self, input_ids, attention_mask, image_hw, class_name_ids=None, cls_indices=None,
                  class_name_embedding_indices=None, token_refer_id=None, refer_embedding_indices=None):
        return SEQ.build_plan(input_ids, attention_mask, self.make_plan_n_img(image_hw), self.num_queries, class_name_ids, cls_indices,
                              class_name_embedding_indices, token_refer_id, refer_embedding_indices)

    def _cached_plan(self, input_ids, attention_mask, image_hw, class_name_ids, cls_indices,
                     class_name_embedding_indices, token_refer_id, refer_embedding_indices):
        """The sequence plan depends only on the prompt (ids / masks / class-name tables) and the image size;
        evaluation loops reuse one prompt for every image, so the device-resident plan is cached by content."""
        key = (tuple(image_hw),) + tuple(_content_key(t) for t in (input_ids, attention_mask, class_name_ids, cls_indices,
                                                              class_name_embedding_indices, token_refer_id,
                                                              refer_embedding_indices))
        return self._lru("_plans", key, lambda: self.make_plan(
            input_ids, attention_mask, image_hw, class_name_ids, cls_indices, class_name_embedding_indices, token_refer_id,
            refer_embedding_indices).to(self.device), self.MAX_PLANS)

    @torch.no_grad()
    def eval_seg(self, input_ids=None, attention_mask=None, past_key_values=None, inputs_embeds=None, labels=None,
                 use_cache=None, output_attentions=None, output_hidden_states=None, images=None, return_dict=None,
                 seg_info=None, class_name_ids=None, class_name_embedding_indices=None, cls_indices=None,
                 token_refer_id=None, refer_embedding_indices=None, is_thing_list=None, region_points=None, vp_images=None,
                 mask_format="dense"):
        """`mask_format`: "dense" (default) returns the reference's results; "rle" adds `instances.pred_masks_rle`, the
        COCO RLE dicts of `instances.pred_masks` encoded on the device (psalm_b200/rle.py), to every result with
        instances - what a COCO evaluator consumes, without copying the dense masks to the host."""
        return self.eval_seg_async(region_points=region_points, vp_images=vp_images, input_ids=input_ids, attention_mask=attention_mask, images=images, seg_info=seg_info,
                                   class_name_ids=class_name_ids, class_name_embedding_indices=class_name_embedding_indices,
                                   cls_indices=cls_indices, token_refer_id=token_refer_id,
                                   refer_embedding_indices=refer_embedding_indices, is_thing_list=is_thing_list,
                                   mask_format=mask_format).result()

    @torch.no_grad()
    def eval_seg_async(self, input_ids=None, attention_mask=None, images=None, seg_info=None, class_name_ids=None,
                       class_name_embedding_indices=None, cls_indices=None, token_refer_id=None,
                       refer_embedding_indices=None, is_thing_list=None, lane=0, region_points=None, vp_images=None,
                       mask_format="dense"):
        """Submit one `eval_seg` call and return a `PendingSeg`; `.result()` gives what `eval_seg` returns.  `lane`
        selects an independent CUDA graph + static output buffers, so that a caller alternating lanes 0 / 1 can finish
        batch k (host merge, read-back) while the device already runs batch k+1.  `region_points`: optional per-sample
        [K,256,2] sample points for <region> prompts (default: drawn like the reference, psalm_b200/region.py).
        `mask_format`: see `eval_seg`; the encoding runs in `result()`."""
        if mask_format not in MASK_FORMATS:
            raise ValueError("mask_format must be one of %s, got %r" % (MASK_FORMATS, mask_format))
        if self.panoptic_on:
            assert is_thing_list is not None, "is_thing_list need to be given"   # llava_phi.py:1337-1339
            self.is_thing_list = is_thing_list
        images_d = self._device_images(images)
        plan = self._cached_plan(input_ids, attention_mask, images.shape[-2:], class_name_ids, cls_indices,
                                 class_name_embedding_indices, token_refer_id, refer_embedding_indices)
        has_regions = plan.region_pos is not None
        if has_regions:   # llava_phi.py:1346-1349: the regions come with the request (seg_info[i]['instances'].region_masks)
            from .region import region_inputs
            pts, img, counts = region_inputs(seg_info, region_points, "region_masks" if vp_images is None else "vp_region_masks")
            assert counts == plan.region_counts, "the munber of <region> tokens and regions needs to be same"   # llava_phi.py:593
            plan = copy.copy(plan)
            plan.region_points, plan.region_image = pts.to(self.device), img.to(self.device)
            if vp_images is not None:
                plan.vp_images = vp_images.to(self.device)
        fused, boxes = self._fused_applies(images.shape[-2:], seg_info)
        if self.use_cuda_graph and not has_regions:   # the number of regions varies per request: eager launches
            out = self.forward_core_graphed(images_d, plan, lane=lane, fuse_post=fused)
        else:
            out = self.forward_core(images_d, plan)
        self._release_staged(images)
        cur = torch.cuda.current_stream(self.device)
        hostvecs = None
        if out.get("post") is not None:   # the integers of the host merge: device -> pinned memory, behind the pass
            if not hasattr(self, "_hostvec_pins"):
                self._hostvec_pins = {}
            hostvecs = []
            for b, d in enumerate(out["post"]):
                hv = d["hostvec"]
                if hv is None:
                    hostvecs.append(None)
                    continue
                k = (lane, b, tuple(hv.shape), hv.dtype)
                pin = self._hostvec_pins.get(k)
                if pin is None:
                    pin = self._hostvec_pins[k] = torch.empty(hv.shape, dtype=hv.dtype, pin_memory=True)
                pin.copy_(hv, non_blocking=True)
                hostvecs.append(pin)
        done = torch.cuda.Event()
        done.record(cur)
        return PendingSeg(self, [(out, hostvecs, getattr(self, "is_thing_list", None))], tuple(images.shape[-2:]), seg_info,
                          boxes, done, (self.object_mask_threshold, self.overlap_threshold), mask_format)

    def _padded(self, image_hw):
        """Size of the padded batch (ImageList.from_tensors(images, 32), llava_phi.py:1400)."""
        d = self.size_divisibility
        return tuple((x + d - 1) // d * d for x in image_hw)

    def _geoms(self, image_hw, seg_info, boxes):
        """Per image (oh, ow, height, width): the un-padded box and the output size."""
        return tuple((box[0], box[1], info.get("height", image_hw[0]), info.get("width", image_hw[1]))
                     for info, box in zip(seg_info, boxes))

    def _routes(self, image_hw, geoms, out=None):
        """Which task heads serve each image: its geometry (`_geoms`) when the fused kernel does - the composed
        up-sample -> crop -> resize unless the geometry is the padded size itself -, None for the torch heads.  `out`:
        forward_core's output; None before the forward, when the class count is not known yet (decided again on `out`)."""
        Hp, Wp = self._padded(image_hw)
        if out is None:
            ps = self.cfg.swin.patch
            Q, ncls, (H4, W4) = self.num_queries, 0, (-(-image_hw[0] // ps), -(-image_hw[1] // ps))
        else:
            cls = out["pred_class_name_logits"]
            Q, ncls, (H4, W4) = out["pred_masks"].shape[1], 0 if cls is None else cls.shape[-1] - 1, out["mask_size"]
        if not (self.fused_postprocess and Q <= PP.FUSED_MAX_QUERIES and ncls <= PP.FUSED_MAX_CLASSES and
                Hp >= 2 * H4 and Wp >= 2 * W4):
            return [None] * len(geoms)
        from . import kernels
        return [g if g == (Hp, Wp, Hp, Wp) or (self.sem_seg_postprocess_before_inference and kernels.postproc_crop_supported(
                    Q, H4, W4, Hp, Wp, *g, PP.FUSED_MAX_CLASSES)) else None
                for g in geoms]

    def _post_device(self, out, image_hw, routes, is_thing_list, obj_thr):
        """Device part of the fused task heads (capturable) for the images `routes` sends to the fused kernel: per image
        the dict `PP.fused_host` finishes, None for the images of the torch heads."""
        idx = [b for b, r in enumerate(routes) if r is not None]
        post = [None] * len(routes)
        if not idx:
            return post
        from . import kernels
        Hp, Wp = self._padded(image_hw)
        H4, W4 = out["mask_size"]
        B, Q = out["pred_masks"].shape[:2]
        pick = lambda t: t if t is None or len(idx) == B else t[idx]   # noqa: E731
        thing = PP.thing_tensor(is_thing_list, self.device) if (self.panoptic_on and self.instance_on) else None
        ds = PP.fused_device_batch(kernels, pick(out["pred_masks"]).view(len(idx), Q, H4, W4), [routes[b][2:] for b in idx],
                                   pick(out["pred_class_name_logits"]), pick(out["pred_SEG_logits"]), thing,
                                   self.semantic_on, self.instance_on, self.panoptic_on, self.referring_on,
                                   self.test_topk_per_image, obj_thr,
                                   crops=[None if routes[b] == (Hp, Wp, Hp, Wp) else (Hp, Wp) + routes[b][:2] for b in idx])
        for b, d in zip(idx, ds):
            post[b] = d
        return post

    def _fused_applies(self, image_hw, seg_info):
        """(fuse_post, boxes): fuse_post is True when every image takes the fused task-head kernel without crop / resize,
        a tuple of per-image (oh, ow, height, width) when the composed up-sample -> crop -> resize kernel applies to all of
        them (the reference's mapper flow: padded 1024^2 input, original-size output), False otherwise (the graph is then
        captured without the task heads instead of running them for nothing)."""
        boxes = [PP.unpadded_box(info["padding_mask"]) for info in seg_info]
        geoms = self._geoms(image_hw, seg_info, boxes)
        Hp, Wp = self._padded(image_hw)
        if all(g == (Hp, Wp, Hp, Wp) for g in geoms):
            return True, boxes
        return (geoms if all(r is not None for r in self._routes(image_hw, geoms)) else False), boxes

    @torch.no_grad()
    def post_process(self, out, image_hw, seg_info, boxes=None, hostvecs=None, is_thing_list=None,
                     object_mask_threshold=None, overlap_threshold=None):
        """llava_phi.py:1395-1472 for EVERY image of the batch.  `boxes`: un-padded (h, w) per image when the
        caller already derived them from the padding masks; `hostvecs`: the fused heads' host vectors when they were
        already copied to (pinned) host memory.  `is_thing_list` and the panoptic thresholds default to the model's
        attributes.  The fused heads' device part runs here unless `out` already holds it for these geometries."""
        if is_thing_list is None:
            is_thing_list = getattr(self, "is_thing_list", None)
        obj_thr = self.object_mask_threshold if object_mask_threshold is None else object_mask_threshold
        ovl_thr = self.overlap_threshold if overlap_threshold is None else overlap_threshold
        with self._precision_scope():
            return self._post_process(out, image_hw, seg_info, boxes, hostvecs, is_thing_list, obj_thr, ovl_thr)

    def _post_process(self, out, image_hw, seg_info, boxes, hostvecs, is_thing_list, obj_thr, ovl_thr):
        Hp, Wp = self._padded(image_hw)
        H4, W4 = out["mask_size"]
        B, Q = out["pred_masks"].shape[:2]
        if boxes is None:
            boxes = [PP.unpadded_box(info["padding_mask"]) for info in seg_info]
        geoms = self._geoms(image_hw, seg_info, boxes)
        post = out.get("post")
        if post is None or out["post_geoms"] != geoms:
            post, hostvecs = self._post_device(out, image_hw, self._routes(image_hw, geoms, out), is_thing_list, obj_thr), None
        pm = out["pred_masks"].view(B, Q, H4, W4)
        mask_pred = None
        results = []
        for b in range(B):
            if post[b] is not None:
                results.append(PP.fused_host(post[b], is_thing_list, ovl_thr,
                                             host=None if hostvecs is None or hostvecs[b] is None else hostvecs[b].numpy()))
                continue
            info = seg_info[b]
            oh, ow, height, width = geoms[b]
            if mask_pred is None:
                mask_pred = F.interpolate(pm.float(), size=(Hp, Wp), mode="bilinear", align_corners=False)
            mp = mask_pred[b]
            r = {}
            if self.sem_seg_postprocess_before_inference:
                mp = PP.sem_seg_postprocess(mp, (oh, ow), height, width)
            cls = out["pred_class_name_logits"][b].float() if out["pred_class_name_logits"] is not None else None
            mp = mp.contiguous()
            sig = mp.sigmoid()   # shared by the task heads below (the reference recomputes it per head)
            tf32 = self.dtype != torch.float32
            if self.semantic_on:
                sem = PP.semantic_inference(cls, mp, sig, tf32)
                if not self.sem_seg_postprocess_before_inference:
                    sem = PP.sem_seg_postprocess(sem, (oh, ow), height, width)
                r["sem_seg"] = sem
            if self.instance_on:
                r["instances"] = PP.instance_inference(cls, mp, self.test_topk_per_image, is_thing_list, self.panoptic_on,
                                                       sig)
            if self.panoptic_on:
                r["panoptic_seg"] = PP.panoptic_inference(cls, mp, is_thing_list, obj_thr, ovl_thr, sig)
            if self.referring_on:
                r["instances"] = PP.seg_instance_inference(out["pred_SEG_logits"][b].float(), mp,
                                                           self.test_topk_per_image, sig)
            if self.region_on:   # llava_phi.py:1457-1466
                r["instances"] = PP.region_inference(out["pred_region_logits"][b].float(), mp, sig)
                gt = getattr(info.get("instances"), "gt_masks", None)   # a session's image may come without them
                if gt is not None:
                    gt = gt.tensor if hasattr(gt, "tensor") else gt
                    r["gt"] = PP.sem_seg_postprocess(gt.to(mp.device).float(), (oh, ow), height, width)
            results.append(r)
        return results


class VideoFrame:
    """Result of one `VideoSession.step`: what eval_davis.py:433-480 computes for the frame.
    labels uint8 [H,W] on the device (`fused_pred_mask`, eval_davis.py:460), query_index int64 [K] and scores fp32 [K]
    (the picked query and its score per object, :443-453), fill_numbers int64 [K], memory_updated (the IoU check of
    :463-480 passed and the frame became the clip's memory; always False without memory)."""

    def __init__(self, labels, query_index, scores, fill_numbers, memory_updated):
        self.labels, self.query_index, self.scores = labels, query_index, scores
        self.fill_numbers, self.memory_updated = fill_numbers, memory_updated


class PendingFrame:
    """Handle of a submitted `VideoSession.step_async`.  `result()` waits for the frame's one small device-to-host copy,
    makes the memory decision and returns the `VideoFrame`.  Its `labels` stay valid until two more frames of the
    session have been submitted."""

    def __init__(self, sess, labels, host, done):
        self.sess, self.labels, self.host, self.done = sess, labels, host, done
        self._frame = None

    def result(self):
        if self._frame is None:
            self._frame = self.sess._finish(self)
        return self._frame


def memory_check(area, inter):
    """eval_davis.py:464-473 on the counts of the kept masks: False when any two objects i != j overlap with
    IoU = |i & j| / |i | j| > 0.4.  An IoU of 0 / 0 (two empty masks) is NaN in numpy and fails no comparison."""
    K = len(area)
    for i in range(K):
        for j in range(K):
            if i != j:
                union = int(area[i]) + int(area[j]) - int(inter[i][j])
                if union > 0 and int(inter[i][j]) / union > 0.4:
                    return False
    return True


class VideoSession:
    """One clip opened by `PSALMForDAVISEval.open_video`: the DAVIS evaluation loop of eval_davis.py:388-480 with its
    state on the device.  The first frame's projector tokens and region masks are kept for the whole clip; each
    `step(images, seg_info)` encodes the frame once (Swin, projector, pixel decoder, decoder memory), pools the K regions
    from the memory frame (the last frame whose prediction passed the IoU check) or from the first frame, runs the prompt
    pass and the region heads, picks one query per object, fuses the label map and keeps the picked masks as the
    candidate memory.  Valid until the next `open_video` / `open_image` on the same lane (a stale session raises
    RuntimeError)."""

    MAX_OBJECTS = 32

    def __init__(self, model, lane, gen, bufs, first_counts, fills, with_memory):
        self.model, self.lane, self.gen, self.bufs = model, lane, gen, bufs
        self.K = len(fills)
        self.first_counts, self.fills, self.with_memory = list(first_counts), fills, bool(with_memory)
        self.mem_counts = None           # set pixels of the memory masks, None until a frame passes the check
        self.pending = None              # the last submitted frame whose memory decision is not made yet
        self.frames = 0
        dev = model.device
        oh, ow, H, W = bufs["geom"]
        hv = bufs["hostvec_len"]
        pin = dev.type == "cuda"
        self._labels = [torch.empty((H, W), dtype=torch.uint8, device=dev) for _ in range(2)]
        self._host = [torch.empty(hv, dtype=torch.int32, pin_memory=pin) for _ in range(2)]

    @torch.no_grad()
    def step(self, images, seg_info):
        return self.step_async(images, seg_info).result()

    @torch.no_grad()
    def step_async(self, images, seg_info):
        """Submit the next frame (images [1,3,H,W], float or uint8, as eval_seg; seg_info: the frame's mapper dict list).
        The frame's image phase is enqueued first; then the previous frame's memory decision is made (its small copy
        is waited for while the device encodes this frame), and the prompt phase follows."""
        m, b = self.model, self.bufs
        m._check_lane(self.lane, self.gen, "stale VideoSession: open_video / open_image was called again on lane %d")
        if images.shape[0] != 1 or len(seg_info) != 1:
            raise ValueError("step takes one frame (got %d)" % images.shape[0])
        if tuple(images.shape[-2:]) != b["image_hw"]:
            raise ValueError("frame size %s differs from the clip's %s" % (tuple(images.shape[-2:]), b["image_hw"]))
        geom = m._geoms(b["image_hw"], seg_info, [PP.unpadded_box(seg_info[0]["padding_mask"])])[0]
        if geom != b["geom"]:
            raise ValueError("frame geometry %s differs from the clip's %s" % (geom, b["geom"]))
        state = m._encode_image(images.to(m.device, non_blocking=True), self.lane)
        if self.pending is not None:
            self.pending.result()
        self._plan_inputs()
        out = m._phase("_video_graphs", (), lambda: m._video_core(state, b), reads=(state, b))
        r = self.frames % 2
        labels, host = self._labels[r], self._host[r]
        labels.copy_(out["labels"])
        host.copy_(out["hostvec"], non_blocking=True)
        done = None
        if m.device.type == "cuda":
            done = torch.cuda.Event()
            done.record(torch.cuda.current_stream(m.device))
        self.pending = PendingFrame(self, labels, host, done)
        self.frames += 1
        return self.pending

    def _plan_inputs(self):
        """Host-planned inputs of the prompt phase: the 256 sample-point indices per region, drawn with the reference's
        calls from the set-pixel counts of the source masks (memory or first frame), and the source slots."""
        from .region import draw_point_indices
        K, b = self.K, self.bufs
        use_mem = self.with_memory and self.mem_counts is not None
        sel = draw_point_indices(self.mem_counts if use_mem else self.first_counts)
        slot = 1 if use_mem else 0
        host = torch.cat([sel.view(-1), torch.arange(slot * K, slot * K + K, dtype=torch.int32),
                          torch.full((K,), slot, dtype=torch.int32), torch.as_tensor(self.fills, dtype=torch.int32)])
        b["inputs"].copy_(host, non_blocking=True)

    def _finish(self, pending):
        K, b = self.K, self.bufs
        if pending.done is not None:
            pending.done.synchronize()
        hv = pending.host.numpy()
        pick = hv[:K].astype("int64")
        score = hv[K:2 * K].copy().view("float32")
        area = hv[2 * K:3 * K]
        inter = hv[3 * K:3 * K + K * K].reshape(K, K)
        counts = hv[3 * K + K * K:4 * K + K * K].tolist()
        updated = False
        if self.with_memory and memory_check(area, inter):
            # promote the candidate (this frame's tokens and kept masks) to the memory slot, in stream order: the next
            # prompt phase, which overwrites the candidate, runs after these copies
            b["src_tok"][1].copy_(b["src_tok"][2])
            b["bits"][K:2 * K].copy_(b["bits"][2 * K:])
            b["prefix"][K:2 * K].copy_(b["prefix"][2 * K:])
            self.mem_counts = counts
            updated = True
        if self.pending is pending:
            self.pending = None
        return VideoFrame(pending.labels, torch.from_numpy(pick), torch.from_numpy(score),
                          torch.as_tensor(self.fills, dtype=torch.int64), updated)


class PSALMForDAVISEval(PSALM):
    """Video-object-segmentation variant (llava_phi.py:1477-2012, builder.py:47 'psalm_video'): the <region> prompts of
    the current frame are pooled from a VISUAL-PROMPT frame (`vp_images`, usually the first frame of the clip) with
    `seg_info[i]['instances'].vp_region_masks`; everything after the sequence splice is PSALM.eval_seg.  The reference's
    `eval_seg` and `eval_video` of this class run the same computation.  `open_video` runs the reference's whole
    per-frame DAVIS loop (eval_davis.py:388-480) as a session."""

    def eval_seg(self, *args, vp_images=None, **kw):
        if vp_images is None:
            raise ValueError("PSALMForDAVISEval needs vp_images (the visual-prompt frames, llava_phi.py:1497)")
        return super().eval_seg(*args, vp_images=vp_images, **kw)

    eval_video = eval_seg

    @torch.no_grad()
    def open_video(self, vp_images, seg_info, input_ids, attention_mask=None, lane=0, with_memory=True):
        """Open a clip: vp_images [1,3,H,W] is the first (visual-prompt) frame, seg_info its mapper dict list with
        `instances.vp_region_masks` [K,H,W] and `instances.vp_fill_number` [K], input_ids / attention_mask the DAVIS
        prompt with K <region> tokens.  The frame is encoded once and its projector tokens kept for the clip.  Returns a
        `VideoSession`; `with_memory` is eval_davis.py's flag.  K <= 32 and fill numbers in 1..255 (the label map is
        uint8), else ValueError."""
        if vp_images.shape[0] != 1 or len(seg_info) != 1:
            raise ValueError("open_video takes one visual-prompt frame (got %d)" % vp_images.shape[0])
        inst = seg_info[0]["instances"]
        masks = inst.vp_region_masks
        masks = (masks.tensor if hasattr(masks, "tensor") else masks).cpu()
        fills = [int(f) for f in torch.as_tensor(inst.vp_fill_number).view(-1).tolist()]
        K = len(fills)
        if not 1 <= K <= VideoSession.MAX_OBJECTS or masks.shape[0] != K:
            raise ValueError("open_video: %d objects with %d region masks (1..%d objects, one mask each)"
                             % (K, masks.shape[0], VideoSession.MAX_OBJECTS))
        if any(not 1 <= f <= 255 for f in fills):
            raise ValueError("open_video: fill numbers must be in 1..255 (the label map is uint8), got %s" % fills)
        image_hw = tuple(vp_images.shape[-2:])
        if tuple(masks.shape[-2:]) != image_hw:
            raise ValueError("open_video: region masks %s are not at the frame size %s" % (tuple(masks.shape[-2:]), image_hw))
        if attention_mask is None:
            attention_mask = torch.ones_like(input_ids, dtype=torch.bool)
        plan = self._cached_plan(input_ids, attention_mask, image_hw, None, None, None, None, None)
        if plan.B != 1 or plan.region_counts != (K,):
            raise ValueError("open_video: the prompt needs one <region> token per object (%d objects, %s tokens)"
                             % (K, plan.region_counts))
        self._region_projector()
        self._region_side(plan.n_img)
        geom = self._geoms(image_hw, seg_info, [PP.unpadded_box(seg_info[0]["padding_mask"])])[0]
        Hpad, Wpad = self._padded(image_hw)
        if geom != (Hpad, Wpad, Hpad, Wpad):
            from . import kernels
            ps = self.cfg.swin.patch
            H4, W4 = -(-image_hw[0] // ps), -(-image_hw[1] // ps)
            if not kernels.postproc_crop_supported(self.num_queries, H4, W4, Hpad, Wpad, *geom, 0):
                raise ValueError("open_video: geometry %s is outside the fused task-head kernel" % (geom,))
        gen = self._open_lane(lane)
        key = (lane, image_hw, K, geom, _content_key(input_ids), _content_key(attention_mask))
        bufs = self._lru("_video_bufs", key, lambda: self._video_buffers(plan, K, image_hw, geom), self.MAX_GRAPHS)
        state = self._encode_image(vp_images.to(self.device, non_blocking=True), lane)
        bufs["src_tok"][0].copy_(state["img_tok"][0])
        self._first_frame_bits(bufs, masks, K)
        return VideoSession(self, lane, gen, bufs, masks.flatten(1).sum(1).tolist(), fills, with_memory)

    def _video_buffers(self, plan, K, image_hw, geom):
        """Device buffers of a clip shape: token slots (0 first frame, 1 memory, 2 candidate), region mask bits in
        three groups of K with the same roles, the host-planned inputs, the Pillow tables of the kept masks."""
        from .image_processor import nearest_pad_tables
        from .region import NUM_SAMPLE_POINT
        dev = self.device
        Hp, Wp = image_hw
        oh, ow, H, W = geom
        P = NUM_SAMPLE_POINT
        rows, cols = nearest_pad_tables(H, W, (oh, ow), (Hp, Wp))
        inputs = torch.zeros(K * P + 3 * K, dtype=torch.int32, device=dev)
        return dict(plan=plan, K=K, image_hw=(Hp, Wp), geom=geom,
                    src_tok=torch.zeros((3, plan.n_img, self.cfg.phi.hidden), dtype=self.dtype, device=dev),
                    bits=torch.zeros((3 * K, Hp, (Wp + 31) // 32), dtype=torch.int32, device=dev),
                    prefix=torch.zeros((3 * K, Hp + 1), dtype=torch.int32, device=dev),
                    count=torch.zeros(3 * K, dtype=torch.int32, device=dev),
                    inputs=inputs, sel=inputs[:K * P].view(K, P), mask_of_region=inputs[K * P:K * P + K],
                    region_image=inputs[K * P + K:K * P + 2 * K], fill=inputs[K * P + 2 * K:],
                    src_row=rows.to(dev), src_col=cols.to(dev), hostvec_len=4 * K + K * K)

    def _first_frame_bits(self, bufs, masks, K):
        """The first frame's region masks (already at the network input size) -> bit slot 0 (identity tables)."""
        from . import kernels
        Hp, Wp = bufs["image_hw"]
        dev = self.device
        kernels.vos_fuse(masks.to(dev, torch.float32).contiguous(), torch.arange(Hp, dtype=torch.int32, device=dev),
                         torch.arange(Wp, dtype=torch.int32, device=dev), bufs["bits"][:K], bufs["prefix"][:K],
                         bufs["count"][:K])

    def _video_core(self, state, bufs):
        """Prompt phase of one frame (capturable): region pooling from the session's token slots, the Phi prefill, the
        heads, the decoder against the frame's memory, the region heads on the fused kernel (pass 1: per-query mask
        scores; pass 2: the K picked masks), the pick, the label map and the candidate memory.  Returns the label map
        and the one int32 vector the host reads: pick [K], score bits [K], area [K], inter [K*K], candidate counts [K]."""
        from . import kernels
        plan, K = bufs["plan"], bufs["K"]
        Hp, Wp = bufs["image_hw"]
        oh, ow, H, W = bufs["geom"]
        Hpad, Wpad = self._padded((Hp, Wp))
        img_tok = state["img_tok"]
        side = self._region_side(img_tok.shape[1])
        bufs["src_tok"][2].copy_(img_tok[0])
        pts = kernels.region_points_gather(bufs["bits"], bufs["prefix"], bufs["sel"], bufs["mask_of_region"], Hp, Wp)
        feat = kernels.region_pool(bufs["src_tok"], pts, bufs["region_image"], side, side)
        embeds = SEQ.materialize_embeds(plan, self.model.embed_tokens, img_tok, self.seg_query, feat)
        hidden = self.model.phi(embeds, plan.attention_mask if plan.any_padding else None)
        seg_q, SEG_emb, cls_emb, rows = self._llm_heads(plan, hidden)
        out = self.predictor.forward_tokens(None, state["ms_sizes"], None, state["mask_size"], seg_q, SEG_emb, cls_emb,
                                            region_embedding_list=[rows], memory=state["mem"])
        H4, W4 = state["mask_size"]
        logits = out["pred_masks"][0].reshape(-1, H4, W4).contiguous()
        crop = None if (oh, ow, H, W) == (Hpad, Wpad, Hpad, Wpad) else (Hpad, Wpad, oh, ow)
        stats = kernels.postproc_fused(logits, H, W, crop=crop)["stats"]
        pick, score = kernels.vos_pick(out["pred_region_logits"][0].contiguous(), stats)
        masks = kernels.postproc_fused(logits, H, W, slot_query=pick, crop=crop)["inst_masks"]
        labels = torch.empty((H, W), dtype=torch.uint8, device=logits.device)
        area = torch.empty(K, dtype=torch.int32, device=logits.device)
        inter = torch.empty((K, K), dtype=torch.int32, device=logits.device)
        kernels.vos_fuse(masks, bufs["src_row"], bufs["src_col"], bufs["bits"][2 * K:], bufs["prefix"][2 * K:],
                         bufs["count"][2 * K:], fill=bufs["fill"], labels=labels, area=area, inter=inter)
        hostvec = torch.cat([pick, score.view(torch.int32), area, inter.view(-1), bufs["count"][2 * K:]])
        return dict(labels=labels, hostvec=hostvec)
