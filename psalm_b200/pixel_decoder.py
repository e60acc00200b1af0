"""Mask2Former pixel decoder (6 x MSDeformAttn encoder + FPN + mask_features), token-major.

Mirrors `MSDeformAttnPixelDecoder.forward_features` (reference mask_decoder/Mask2Former_Simplify/
modeling/pixel_decoder/msdeformattn.py:268-315), the encoder (:136-164, :89-95, :57-66) and
`MSDeformAttn.forward` (ops/modules/ms_deform_attn.py:82-124).  Differences from the reference:
  * feature maps are [B, H*W, C] (C contiguous): 1x1 convolutions are plain GEMMs and mask_features
    comes out K-major for the mask-projection kernel;
  * sampling_offsets and attention_weights are ONE GEMM (288 outputs); softmax, reference points,
    location arithmetic and the bilinear gather run in ONE kernel (psalm_msda_encoder_fused) on a
    head-major value tensor — `sampling_locations` (16.5 MB) and `attention_weights` (8.3 MB) per layer
    never exist, nor does the reference's fp32 up-cast copy of `value` (ms_deform_attn.py:113-115);
  * sine position embeddings are input independent and cached per (H, W) (the reference recomputes
    them 6x per image, position_encoding.py:29-52).
"""
import math

import torch
import torch.nn.functional as F

from . import kernels
from .layout import MaskConfig

_POS_CACHE = {}


def position_embedding_sine_tokens(H, W, device, num_pos_feats=128, temperature=10000.0):
    """PositionEmbeddingSine(normalize=True) for an unmasked H x W map -> [H*W, 256] fp32, cached.
    (transformer_decoder/position_encoding.py:29-52)"""
    key = (H, W, str(device))
    if key not in _POS_CACHE:
        y = torch.arange(1, H + 1, dtype=torch.float32).view(H, 1).expand(H, W)
        x = torch.arange(1, W + 1, dtype=torch.float32).view(1, W).expand(H, W)
        eps, scale = 1e-6, 2 * math.pi
        y = y / (float(H) + eps) * scale
        x = x / (float(W) + eps) * scale
        dim_t = torch.arange(num_pos_feats, dtype=torch.float32)
        dim_t = temperature ** (2 * torch.div(dim_t, 2, rounding_mode="floor") / num_pos_feats)
        px = x[:, :, None] / dim_t
        py = y[:, :, None] / dim_t
        px = torch.stack((px[:, :, 0::2].sin(), px[:, :, 1::2].cos()), dim=3).flatten(2)
        py = torch.stack((py[:, :, 0::2].sin(), py[:, :, 1::2].cos()), dim=3).flatten(2)
        _POS_CACHE[key] = torch.cat((py, px), dim=2).view(H * W, 2 * num_pos_feats).to(device)
    return _POS_CACHE[key]


def group_norm_tokens(x, weight, bias, groups=32, eps=1e-5):
    """GroupNorm(32) of a token-major map [B, HW, C] (statistics over HW x C/groups), fp32 statistics."""
    B, N, C = x.shape
    xf = x.float().view(B, N, groups, C // groups)
    mean = xf.mean(dim=(1, 3), keepdim=True)
    var = xf.var(dim=(1, 3), unbiased=False, keepdim=True)
    y = ((xf - mean) * torch.rsqrt(var + eps)).view(B, N, C)
    return (y * weight.float() + bias.float()).to(x.dtype)


class MSDeformAttnPixelDecoder:
    def __init__(self, sd, prefix="pixel_decoder.", cfg=MaskConfig(), dtype=torch.bfloat16, device="cuda"):
        self.cfg, self.dtype, self.device = cfg, dtype, device
        cv = lambda t: t.to(device=device, dtype=dtype).contiguous()  # noqa: E731
        g = lambda k: sd[prefix + k]  # noqa: E731
        w = {}
        for i in range(cfg.enc_levels):  # res5, res4, res3
            w["ip%d.w" % i] = cv(g("input_proj.%d.0.weight" % i).flatten(1))
            w["ip%d.b" % i] = cv(g("input_proj.%d.0.bias" % i))
            w["ip%d.gw" % i], w["ip%d.gb" % i] = cv(g("input_proj.%d.1.weight" % i)), cv(g("input_proj.%d.1.bias" % i))
        self.level_embed = g("transformer.level_embed").float().to(device)
        for i in range(cfg.enc_layers):
            p = "transformer.encoder.layers.%d." % i
            a = p + "self_attn."
            # offsets (192) and logits (96) as one GEMM: rows [offsets | logits] = the fused kernel's layout
            w["e%d.ow.w" % i] = cv(torch.cat([g(a + "sampling_offsets.weight"), g(a + "attention_weights.weight")], 0))
            w["e%d.ow.b" % i] = cv(torch.cat([g(a + "sampling_offsets.bias"), g(a + "attention_weights.bias")], 0))
            for n, k in (("vp", "value_proj"), ("op", "output_proj")):
                w["e%d.%s.w" % (i, n)], w["e%d.%s.b" % (i, n)] = cv(g(a + k + ".weight")), cv(g(a + k + ".bias"))
            for n in ("norm1", "norm2", "linear1", "linear2"):
                w["e%d.%s.w" % (i, n)], w["e%d.%s.b" % (i, n)] = cv(g(p + n + ".weight")), cv(g(p + n + ".bias"))
        w["mf.w"], w["mf.b"] = cv(g("mask_features.weight").flatten(1)), cv(g("mask_features.bias"))
        w["ad.w"], w["ad.b"] = cv(g("adapter_1.0.weight").flatten(1)), cv(g("adapter_1.0.bias"))
        w["ad.gw"], w["ad.gb"] = cv(g("adapter_1.1.weight")), cv(g("adapter_1.1.bias"))
        w["l1.w"] = g("layer_1.0.weight").to(device=device, dtype=dtype).contiguous(memory_format=torch.channels_last)
        w["l1.b"] = cv(g("layer_1.0.bias"))
        w["l1.gw"], w["l1.gb"] = cv(g("layer_1.1.weight")), cv(g("layer_1.1.bias"))
        self.w = w

    def forward_features(self, features):
        """Reference surface (msdeformattn.py:268): dict res2..res5 of NCHW maps ->
        (mask_features NCHW, encoder res5-level NCHW, [3 multi-scale NCHW maps]); views of token maps."""
        toks, sizes = [], []
        for k in ("res2", "res3", "res4", "res5"):
            f = features[k]
            B, C, H, W = f.shape
            toks.append(f.permute(0, 2, 3, 1).reshape(B, H * W, C).to(self.dtype))
            sizes.append((H, W))
        mf, ms, ms_sizes = self.forward_tokens(toks, sizes)
        nchw = lambda t, hw: t.view(t.shape[0], hw[0], hw[1], t.shape[2]).permute(0, 3, 1, 2)  # noqa: E731
        return nchw(mf, sizes[0]), nchw(ms[0], ms_sizes[0]), [nchw(t, s) for t, s in zip(ms, ms_sizes)]

    def forward_tokens(self, toks, sizes):
        """toks: [res2,res3,res4,res5] token-major [B,HW,C]; sizes: [(H,W)] ->
        (mask_features [B,H2*W2,256], [tokens of the 32^2/64^2/128^2-level maps], their sizes)."""
        cfg, w = self.cfg, self.w
        B = toks[0].shape[0]
        srcs, poss, shapes = [], [], []
        for i, li in enumerate((3, 2, 1)):  # res5, res4, res3 (msdeformattn.py:272-276)
            x = F.linear(toks[li], w["ip%d.w" % i], w["ip%d.b" % i])
            srcs.append(kernels.group_norm_tokens(x, w["ip%d.gw" % i], w["ip%d.gb" % i]))
            H, W = sizes[li]
            shapes.append((H, W))
            pe = position_embedding_sine_tokens(H, W, self.device).to(self.dtype)   # .to(x.dtype) at :276
            poss.append((pe.float() + self.level_embed[i]).to(self.dtype) if self.dtype == torch.float32
                        else (pe + self.level_embed[i].to(self.dtype)))
        src = torch.cat(srcs, 1).contiguous()
        pos = torch.cat(poss, 0).unsqueeze(0)
        S = src.shape[1]
        starts, acc = [], 0
        for h_, w_ in shapes:
            starts.append(acc)
            acc += h_ * w_
        M, D = cfg.nheads, cfg.hidden // cfg.nheads
        # (src + pos) W^T + b = src W^T + (pos W^T + b): the position term is input independent, so it is
        # projected once per (shapes, batch) and enters the GEMM as its additive C matrix; the per-layer
        # broadcast add and the `q` tensor (ms_deform_attn.py:57-58 with_pos_embed) do not exist
        # keyed by (shapes, batch) and never evicted: captured CUDA graphs hold these device pointers, so an entry
        # must stay alive (and unmoved) for as long as any graph of that size may be replayed
        pkey = (tuple(shapes), B)
        if not hasattr(self, "_pos_ow_cache"):
            self._pos_ow_cache = {}
        pos_ow = self._pos_ow_cache.get(pkey)
        if pos_ow is None:
            p32 = pos[0].float()
            pos_ow = [(p32 @ w["e%d.ow.w" % i].float().t() + w["e%d.ow.b" % i].float()).to(self.dtype)
                      .repeat(B, 1).contiguous() for i in range(cfg.enc_layers)]
            self._pos_ow_cache[pkey] = pos_ow
        for i in range(cfg.enc_layers):
            ow = torch.addmm(pos_ow[i], src.view(B * S, -1), w["e%d.ow.w" % i].t()).view(B, S, -1)
            if D == 32 and kernels.linear_fused_supported(src, w["e%d.vp.w" % i], "head_major", S):
                # value_proj with the head-major store in the GEMM epilogue (csrc/gemm_tc5.cu): no transposing copy
                value_hm = kernels.linear_fused(src, w["e%d.vp.w" % i], w["e%d.vp.b" % i], "head_major", S)
            else:
                value = F.linear(src, w["e%d.vp.w" % i], w["e%d.vp.b" % i])
                value_hm = value.view(B, S, M, D).permute(0, 2, 1, 3).contiguous()
            a = kernels.timed_msda(kernels.msda_encoder_fused, value_hm, ow.contiguous(), shapes, starts, cfg.enc_points)
            kernels._count()
            src = kernels.add_layer_norm(src, w["e%d.norm1.w" % i], w["e%d.norm1.b" % i],
                                         r1=F.linear(a, w["e%d.op.w" % i], w["e%d.op.b" % i]))
            f = F.linear(kernels.linear_act(src, w["e%d.linear1.w" % i], w["e%d.linear1.b" % i], "relu"),
                         w["e%d.linear2.w" % i], w["e%d.linear2.b" % i])
            src = kernels.add_layer_norm(src, w["e%d.norm2.w" % i], w["e%d.norm2.b" % i], r1=f)
        outs = [t.contiguous() for t in torch.split(src, [h_ * w_ for h_, w_ in shapes], dim=1)]
        # FPN level on res2 (msdeformattn.py:300-309)
        H2, W2 = sizes[0]
        cur = kernels.group_norm_tokens(F.linear(toks[0], w["ad.w"], w["ad.b"]), w["ad.gw"], w["ad.gb"], relu=True)
        Hl, Wl = shapes[-1]
        if self.dtype == torch.float32:
            up = kernels.bilinear_tokens(outs[-1], Hl, Wl, H2, W2)   # fp32 math, rounded to dtype like `.to(x.dtype)`
            y = cur + up
        else:   # 16-bit storage: the up-sampled map is added in the resampling kernel (one pass instead of three)
            y = kernels.bilinear_tokens(outs[-1], Hl, Wl, H2, W2, out=cur, accumulate=True)
        y = y.view(B, H2, W2, cfg.hidden).permute(0, 3, 1, 2)   # channels-last NCHW view
        # the conv runs without its bias (a separate broadcast-add pass in cuDNN); GroupNorm adds it in-kernel
        y = F.conv2d(y, w["l1.w"], None, padding=1).permute(0, 2, 3, 1).reshape(B, H2 * W2, cfg.hidden)
        y = kernels.group_norm_tokens(y.contiguous(), w["l1.gw"], w["l1.gb"], relu=True, pre_bias=w["l1.b"])
        mask_features = F.linear(y, w["mf.w"], w["mf.b"])
        return mask_features, outs, shapes
