"""Masked-attention transformer decoder + prediction heads, batch-first, token-major.

Mirrors `MultiScaleMaskedTransformerDecoderForOPTPreTrain.forward_woconcat`
(reference transformer_decoder/mask2former_transformer_decoder.py:596-693) and
`forward_prediction_heads` (:695-762).  Differences from the reference:
  * masked cross-attention and the 100x100 query self-attention are one fused kernel each
    (psalm_cross_attention) working on a PACKED BIT mask (1 bit / key, shared by the 8 heads) instead of
    nn.MultiheadAttention with a float -inf mask of shape [B*8, 100, HW] and materialised probabilities;
  * the 9 intermediate prediction heads only feed the next attention mask (:668-680; aux outputs are
    unused at inference, llava_phi.py:1395-1398).  Bilinear interpolation and the mask einsum are both
    linear, so  interp(einsum(mask_embed, F)) == einsum(mask_embed, interp(F)):  we interpolate
    mask_features to the three target sizes ONCE per image and each intermediate head is a
    [100 x 256] x [256 x HW_l] projection + sign test, instead of ten full-resolution einsums of which
    nine are thresholded and thrown away (236 MB of logits per image in the reference);
  * `(sigmoid(x) < 0.5)` is `x < 0`; fully blocked rows are opened by a per-row flag (:647).
"""
import torch
import torch.nn.functional as F

from . import kernels
from .layout import MaskConfig
from .pixel_decoder import position_embedding_sine_tokens


class MultiScaleMaskedTransformerDecoderForOPTPreTrain:
    def __init__(self, sd, prefix="predictor.", cfg=MaskConfig(), dtype=torch.bfloat16, device="cuda"):
        self.cfg, self.dtype, self.device = cfg, dtype, device
        cv = lambda t: t.to(device=device, dtype=dtype).contiguous()  # noqa: E731
        g = lambda k: sd[prefix + k]  # noqa: E731
        w = {}
        H = cfg.hidden
        for i in range(cfg.dec_layers):
            for kind, attn, tag in (("cross", "multihead_attn", "x"), ("self", "self_attn", "s")):
                p = "transformer_%s_attention_layers.%d." % (kind, i)
                W, b = g(p + attn + ".in_proj_weight"), g(p + attn + ".in_proj_bias")
                for j, n in enumerate("qkv"):
                    w["%s%d.%s.w" % (tag, i, n)] = cv(W[j * H:(j + 1) * H])
                    w["%s%d.%s.b" % (tag, i, n)] = cv(b[j * H:(j + 1) * H])
                w["%s%d.o.w" % (tag, i)], w["%s%d.o.b" % (tag, i)] = cv(g(p + attn + ".out_proj.weight")), cv(g(p + attn + ".out_proj.bias"))
                w["%s%d.n.w" % (tag, i)], w["%s%d.n.b" % (tag, i)] = cv(g(p + "norm.weight")), cv(g(p + "norm.bias"))
            p = "transformer_ffn_layers.%d." % i
            for n in ("linear1", "linear2", "norm"):
                w["f%d.%s.w" % (i, n)], w["f%d.%s.b" % (i, n)] = cv(g(p + n + ".weight")), cv(g(p + n + ".bias"))
        # K (and V) projections of the decoder layers that share a feature level (layers li, li+3, li+6 read the same
        # memory, :642-650) as ONE weight matrix per level: 2 x 3 GEMMs per image instead of 2 x 9
        for li in range(3):
            layers = list(range(li, cfg.dec_layers, 3))
            for n in "kv":
                w["x%s_all%d.w" % (n, li)] = torch.cat([w["x%d.%s.w" % (i, n)] for i in layers], 0).contiguous()
                w["x%s_all%d.b" % (n, li)] = torch.cat([w["x%d.%s.b" % (i, n)] for i in layers], 0).contiguous()
        w["dn.w"], w["dn.b"] = cv(g("decoder_norm.weight")), cv(g("decoder_norm.bias"))
        self.query_embed = cv(g("query_embed.weight"))      # forward_woconcat uses query_embed (:619)
        self.level_embed = cv(g("level_embed.weight"))
        heads = [("mask_embed", 3), ("SEG_proj", 2), ("CLASS_proj", 2)]
        if prefix + "REGION_proj.layers.0.weight" in sd:    # optional in the checkpoint contract (loader.py)
            heads.append(("REGION_proj", 2))
        for name, n in heads:
            for j in range(n):
                w["%s.%d.w" % (name, j)] = cv(g("%s.layers.%d.weight" % (name, j)))
                w["%s.%d.b" % (name, j)] = cv(g("%s.layers.%d.bias" % (name, j)))
        self.w = w

    def _mlp(self, name, n, x):
        for j in range(n):
            if j < n - 1:
                x = kernels.linear_act(x, self.w["%s.%d.w" % (name, j)], self.w["%s.%d.b" % (name, j)], "relu")
            else:
                x = F.linear(x, self.w["%s.%d.w" % (name, j)], self.w["%s.%d.b" % (name, j)])
        return x

    def _heads_common(self, output):
        dec = kernels.add_layer_norm(output.contiguous(), self.w["dn.w"], self.w["dn.b"])
        return dec, self._mlp("mask_embed", 3, dec)

    # reference-surface entry: NCHW maps in, dict out (mask2former_transformer_decoder.py:488,684-692)
    def __call__(self, x, mask_features, mask=None, seg_query=None, SEG_embedding=None, class_name_embedding=None,
                 region_embedding_list=None):
        sizes = [tuple(t.shape[-2:]) for t in x]
        toks = [t.permute(0, 2, 3, 1).reshape(t.shape[0], -1, t.shape[1]).to(self.dtype).contiguous() for t in x]
        B, C, H4, W4 = mask_features.shape
        mf = mask_features.permute(0, 2, 3, 1).reshape(B, H4 * W4, C).to(self.dtype).contiguous()
        out = self.forward_tokens(toks, sizes, mf, (H4, W4), seg_query, SEG_embedding, class_name_embedding,
                                  region_embedding_list=region_embedding_list)
        out["pred_masks"] = out["pred_masks"].view(B, -1, H4, W4)
        out["aux_outputs"] = []
        return out

    def _fused_kv(self, Q, Hd):
        # 16-bit storage: all K / V projections of a level up front (one GEMM each), consumed as row-strided views by
        # the TMA-fed kernel; fp32 storage keeps the per-layer projections + the SIMT kernel
        return self.dtype != torch.float32 and Hd == 256 and self.cfg.nheads == 8 and Q <= 112

    def memory(self, ms_tokens, ms_sizes, mask_features, mf_size, Q=None):
        """The query-independent part of forward_tokens for images [B]: the K / V projections of the three levels (16-bit
        storage) or their inputs (fp32), and mask_features pooled to the three attention-mask sizes.  A memory of ONE
        image serves any number of query sets (forward_tokens(..., memory=...), the prompts of one image)."""
        cfg, w = self.cfg, self.w
        Hd = ms_tokens[0].shape[-1]
        Q = cfg.num_queries if Q is None else Q
        B = ms_tokens[0].shape[0]
        H4, W4 = mf_size
        mem = dict(B=B, fused_kv=self._fused_kv(Q, Hd), mask_features=mask_features)
        srcs, kins = [], []
        if not mem["fused_kv"]:
            for i in range(3):  # (:607-614); input_proj is the identity (in_channels == hidden_dim, :475-479)
                Hl, Wl = ms_sizes[i]
                pos = position_embedding_sine_tokens(Hl, Wl, self.device).to(self.dtype)
                src = ms_tokens[i] + self.level_embed[i]
                srcs.append(src)
                kins.append(src + pos)
        # attention-mask sources: mask_features interpolated once to each target size (see module docstring)
        mem["pooled"] = [kernels.bilinear_tokens(mask_features, H4, W4, hl, wl) for hl, wl in ms_sizes]
        mem["srcs"], mem["kins"] = srcs, kins
        if mem["fused_kv"]:
            # K = (x + level_embed + pos) Wk^T + bk = x Wk^T + [(level_embed + pos) Wk^T + bk] and
            # V = (x + level_embed) Wv^T + bv = x Wv^T + [Wv level_embed + bv]: the bracketed terms do not depend on the
            # input, so they are projected once per (sizes, batch) and enter the GEMMs as the additive C matrix / the bias;
            # the `src` and `src + pos` tensors (:607-614, six passes over the multi-scale maps) do not exist.
            # Never evicted: captured CUDA graphs hold these device pointers.
            ckey = (tuple(ms_sizes), B)
            if not hasattr(self, "_kv_const"):
                self._kv_const = {}
            kvc = self._kv_const.get(ckey)
            if kvc is None:
                posk, vb = [], []
                for li in range(3):
                    Hl, Wl = ms_sizes[li]
                    pe = position_embedding_sine_tokens(Hl, Wl, self.device).float() + self.level_embed[li].float()
                    pk = pe @ w["xk_all%d.w" % li].float().t() + w["xk_all%d.b" % li].float()
                    posk.append(pk.to(self.dtype).repeat(B, 1).contiguous())
                    vb.append((w["xv_all%d.b" % li].float() + w["xv_all%d.w" % li].float() @ self.level_embed[li].float())
                              .to(self.dtype).contiguous())
                kvc = self._kv_const[ckey] = (posk, vb)
            posk, vb = kvc
            mem["k_all"] = [torch.addmm(posk[li], ms_tokens[li].reshape(-1, Hd), w["xk_all%d.w" % li].t()).view(B, -1, 3 * Hd)
                            for li in range(3)]
            mem["v_all"] = [F.linear(ms_tokens[li], w["xv_all%d.w" % li], vb[li]) for li in range(3)]
        return mem

    def forward_tokens(self, ms_tokens, ms_sizes, mask_features, mf_size, seg_query, SEG_embedding=None,
                       class_name_embedding=None, return_trace=False, hooks=None, region_embedding_list=None, memory=None):
        """ms_tokens: 3 maps [B,HW_l,256] (32^2,64^2,128^2 levels); mask_features [B,H4*W4,256];
        seg_query [B,Q,256].  Returns dict(pred_masks [B,Q,H4*W4], pred_class_name_logits, pred_SEG_logits).
        `memory`: the result of `memory(...)` for these maps (ms_tokens / mask_features are then not read); a memory of
        one image with B query sets runs the B sets against that image.
        `hooks` (tests only, oracle/parity.py): an object whose before_layer(i, output, bits, row_open, mask_for) may
        substitute the decoder state / attention mask entering layer i (layer-wise teacher forcing) and whose
        after_layer(i, output) observes the state leaving it."""
        cfg, w = self.cfg, self.w
        B, Q, Hd = seg_query.shape
        nh = cfg.nheads
        if memory is None:
            memory = self.memory(ms_tokens, ms_sizes, mask_features, mf_size, Q)
        fused_kv = memory["fused_kv"]
        if fused_kv != self._fused_kv(Q, Hd):
            raise ValueError("memory was prepared for another query shape")
        shared = memory["B"] != B
        if shared and memory["B"] != 1:
            raise ValueError("a memory of %d images cannot serve %d query sets" % (memory["B"], B))

        def per_set(t):
            # one image's memory for B query sets: 16-bit kernels read stride-0 `expand` views; the fp32 parity path
            # materialises copies where its kernels need dense batches (psalm_cross_attention has no batch stride)
            if not shared:
                return t
            return t.expand(B, *t.shape[1:]) if fused_kv else t.expand(B, *t.shape[1:]).contiguous()

        pooled = [per_set(t) for t in memory["pooled"]]
        mask_features = per_set(memory["mask_features"])
        srcs, kins = memory["srcs"], memory["kins"]
        if fused_kv:
            k_all, v_all = [per_set(t) for t in memory["k_all"]], [per_set(t) for t in memory["v_all"]]
        qpos = self.query_embed.unsqueeze(0)
        output = seg_query.to(self.dtype).contiguous()
        trace = []

        def mask_for(level, out_):
            _, me = self._heads_common(out_)
            if return_trace:
                trace.append(kernels.mask_logits(me.contiguous(), pooled[level], out_dtype=torch.float32))
            return kernels.mask_bits(me.contiguous(), pooled[level])

        qc = None
        if fused_kv:
            # (output + query_pos) W^T + b = output W^T + (query_pos W^T + b): the position terms of the cross-attention
            # query and of the self-attention query / key do not depend on the input; they enter the GEMMs as the additive
            # C matrix (no `output + query_pos` passes), and the self-attention K and V projections share one GEMM whose
            # halves the attention kernel reads as row-strided views.  Never evicted: CUDA graphs hold these pointers.
            if not hasattr(self, "_q_const"):
                self._q_const = {}
            qc = self._q_const.get(B)
            if qc is None:
                qp = self.query_embed.float()
                qc = []
                for i in range(cfg.dec_layers):
                    lin = lambda n: qp @ w[n + ".w"].float().t() + w[n + ".b"].float()   # noqa: E731
                    cx = lin("x%d.q" % i).to(self.dtype).repeat(B, 1).contiguous()
                    cs = lin("s%d.q" % i).to(self.dtype).repeat(B, 1).contiguous()
                    ckv = torch.cat([lin("s%d.k" % i), w["s%d.v.b" % i].float().expand(Q, -1)], 1)
                    wkv = torch.cat([w["s%d.k.w" % i], w["s%d.v.w" % i]], 0).contiguous()
                    qc.append((cx, cs, ckv.to(self.dtype).repeat(B, 1).contiguous(), wkv))
                self._q_const[B] = qc
        bits, row_open = mask_for(0, output)
        for i in range(cfg.dec_layers):
            li = i % 3
            if hooks is not None:
                output, bits, row_open = hooks.before_layer(i, output, bits, row_open, lambda o_, lv=li: mask_for(lv, o_))
            # masked cross-attention (:93-105): q = tgt + query_pos, k = memory + pos, v = memory
            if fused_kv:
                q = torch.addmm(qc[i][0], output.reshape(-1, Hd), w["x%d.q.w" % i].t()).view(B, Q, Hd)
            else:
                q = F.linear(output + qpos, w["x%d.q.w" % i], w["x%d.q.b" % i])
            if fused_kv:
                j = i // 3
                k, v = k_all[li][:, :, j * Hd:(j + 1) * Hd], v_all[li][:, :, j * Hd:(j + 1) * Hd]
                a = kernels.timed("masked_cross_attention_%d" % k.shape[1], kernels.masked_cross_attention, q, k, v,
                                  bits, row_open, nh)
            else:
                k = per_set(F.linear(kins[li], w["x%d.k.w" % i], w["x%d.k.b" % i]))
                v = per_set(F.linear(srcs[li], w["x%d.v.w" % i], w["x%d.v.b" % i]))
                a = kernels.timed("masked_cross_attention_%d" % k.shape[1], kernels.cross_attention, q, k, v, bits,
                                  row_open, nh)
            output = kernels.add_layer_norm(output, w["x%d.n.w" % i], w["x%d.n.b" % i],
                                            r1=F.linear(a, w["x%d.o.w" % i], w["x%d.o.b" % i]))
            # query self-attention (:35-45): q = k = tgt + query_pos, v = tgt
            if fused_kv:
                o2 = output.reshape(-1, Hd)
                q = torch.addmm(qc[i][1], o2, w["s%d.q.w" % i].t()).view(B, Q, Hd)
                kv = torch.addmm(qc[i][2], o2, qc[i][3].t()).view(B, Q, 2 * Hd)
                a = kernels.masked_cross_attention(q, kv[:, :, :Hd], kv[:, :, Hd:], None, None, nh)
            else:
                xq = output + qpos
                q = F.linear(xq, w["s%d.q.w" % i], w["s%d.q.b" % i])     # three contiguous outputs: no slicing copies
                k = F.linear(xq, w["s%d.k.w" % i], w["s%d.k.b" % i])
                v = F.linear(output, w["s%d.v.w" % i], w["s%d.v.b" % i])
                a = kernels.cross_attention(q, k, v, None, None, nh, splits=1)
            output = kernels.add_layer_norm(output, w["s%d.n.w" % i], w["s%d.n.b" % i],
                                            r1=F.linear(a, w["s%d.o.w" % i], w["s%d.o.b" % i]))
            # FFN (:158-162)
            f = F.linear(kernels.linear_act(output, w["f%d.linear1.w" % i], w["f%d.linear1.b" % i], "relu"),
                         w["f%d.linear2.w" % i], w["f%d.linear2.b" % i])
            output = kernels.add_layer_norm(output, w["f%d.norm.w" % i], w["f%d.norm.b" % i], r1=f)
            if hooks is not None:
                hooks.after_layer(i, output)
            if i < cfg.dec_layers - 1:
                bits, row_open = mask_for((i + 1) % 3, output)
        # final prediction heads (:695-750) — the only ones whose outputs leave the decoder
        dec, me = self._heads_common(output)
        out = dict(pred_SEG_logits=None, pred_class_name_logits=None, pred_region_logits=None)
        if region_embedding_list is not None:   # [K_b, Q] per sample = region_embedding . REGION_proj(decoder_output) (:737-745)
            if "REGION_proj.0.w" not in w:
                raise KeyError("region prompts need predictor.REGION_proj.* in the checkpoint")
            dr = self._mlp("REGION_proj", 2, dec)
            out["pred_region_logits"] = [re.to(self.dtype) @ dr[b].t() for b, re in enumerate(region_embedding_list)]
        if SEG_embedding is not None:
            out["pred_SEG_logits"] = torch.bmm(self._mlp("SEG_proj", 2, dec), SEG_embedding.to(self.dtype).transpose(1, 2))
        if class_name_embedding is not None:
            out["pred_class_name_logits"] = torch.bmm(self._mlp("CLASS_proj", 2, dec),
                                                      class_name_embedding.to(self.dtype).transpose(1, 2))
        out["pred_masks"] = kernels.timed("mask_projection", kernels.mask_logits, me.contiguous(), mask_features)
        if return_trace:
            out["trace_pooled_logits"] = trace
        return out
