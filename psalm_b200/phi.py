"""Phi-1.5 prefill for the PSALM hot path (no autoregressive decode: eval_seg runs ONE causal prefill
over [text | image tokens | class names | 100 seg queries], reference llava_phi.py:1354-1363).

Restates transformers' PhiModel / PhiDecoderLayer / PhiAttention (third-party, pinned 4.36.2 by the
reference, pyproject.toml:27): LN -> (attention || MLP) -> sum + residual, partial rotary on the first
half of each 64-wide head, fp32 softmax, gelu_new, final LayerNorm.  Q/K/V projections are one fused
library GEMM; rotary and the causal attention are hand-written kernels (psalm_rotary_inplace,
psalm_causal_attention); lm_head is never evaluated on this path."""
import torch
import torch.nn.functional as F

from . import kernels
from .layout import PhiConfig


class PhiModel:
    def __init__(self, sd, prefix="model.", cfg=PhiConfig(), dtype=torch.bfloat16, device="cuda"):
        self.cfg, self.dtype, self.device = cfg, dtype, device
        cv = lambda t: t.to(device=device, dtype=dtype).contiguous()  # noqa: E731
        w = {}
        self.embed_tokens = cv(sd[prefix + "embed_tokens.weight"])
        for i in range(cfg.layers):
            p = "%slayers.%d." % (prefix, i)
            a = p + "self_attn."
            w["%d.qkv.w" % i] = cv(torch.cat([sd[a + "q_proj.weight"], sd[a + "k_proj.weight"], sd[a + "v_proj.weight"]], 0))
            w["%d.qkv.b" % i] = cv(torch.cat([sd[a + "q_proj.bias"], sd[a + "k_proj.bias"], sd[a + "v_proj.bias"]], 0))
            w["%d.dense.w" % i], w["%d.dense.b" % i] = cv(sd[a + "dense.weight"]), cv(sd[a + "dense.bias"])
            w["%d.fc1.w" % i], w["%d.fc1.b" % i] = cv(sd[p + "mlp.fc1.weight"]), cv(sd[p + "mlp.fc1.bias"])
            w["%d.fc2.w" % i], w["%d.fc2.b" % i] = cv(sd[p + "mlp.fc2.weight"]), cv(sd[p + "mlp.fc2.bias"])
            w["%d.ln.w" % i], w["%d.ln.b" % i] = cv(sd[p + "input_layernorm.weight"]), cv(sd[p + "input_layernorm.bias"])
        w["fln.w"], w["fln.b"] = cv(sd[prefix + "final_layernorm.weight"]), cv(sd[prefix + "final_layernorm.bias"])
        self.w = w
        self._rope = {}

    def rope_tables(self, T):
        """cos/sin [T, rd/2] fp32 (PhiRotaryEmbedding: inv_freq = theta^(-2i/rd), positions 0..T-1)."""
        if T not in self._rope:
            cfg = self.cfg
            rd = int(cfg.head_dim * cfg.rotary_frac)
            inv = 1.0 / (cfg.rope_theta ** (torch.arange(0, rd, 2, dtype=torch.int64).float() / rd))
            fr = torch.arange(T).float()[:, None] * inv[None, :]
            self._rope[T] = (fr.cos().contiguous().to(self.device), fr.sin().contiguous().to(self.device))
        return self._rope[T]

    def __call__(self, inputs_embeds, attention_mask=None):
        return self.forward(inputs_embeds, attention_mask)

    def forward(self, inputs_embeds, attention_mask=None, cache=None):
        """inputs_embeds [B,T,C]; attention_mask [B,T] (True/1 = real token) or None -> last_hidden_state.
        `cache` (generate.PagedKVCache): the rotary-applied K / V rows of every layer are also written to its pages."""
        cfg, w = self.cfg, self.w
        B, T, C = inputs_embeds.shape
        nh, hd = cfg.heads, cfg.head_dim
        rd = int(hd * cfg.rotary_frac)
        cos, sin = self.rope_tables(T)
        kv = None
        if attention_mask is not None:
            kv = attention_mask.to(device=self.device, dtype=torch.uint8).contiguous()
        h = inputs_embeds.contiguous()
        a = f = None
        for i in range(cfg.layers):
            if a is None:
                x = kernels.add_layer_norm(h, w["%d.ln.w" % i], w["%d.ln.b" % i], cfg.eps)
            else:  # h = attn + mlp + residual of the previous layer, fused with this layer's input_layernorm
                h, x = kernels.add_layer_norm(h, w["%d.ln.w" % i], w["%d.ln.b" % i], cfg.eps, r1=a, r2=f, return_sum=True)
            qkv = F.linear(x, w["%d.qkv.w" % i], w["%d.qkv.b" % i]).view(B, T, 3, nh, hd)
            kernels.rotary_inplace(qkv, cos, sin, B, T, nh, hd, rd)
            if cache is not None:
                kernels.kv_cache_write(qkv, cache.k[i], cache.v[i], cache.block_table, cache.seq_lens)
            a = kernels.timed("causal_attention", kernels.causal_attention, qkv, kv, B, T, nh, hd)
            a = F.linear(a, w["%d.dense.w" % i], w["%d.dense.b" % i])
            f = self._fc1_gelu(x, i)
            f = F.linear(f, w["%d.fc2.w" % i], w["%d.fc2.b" % i])
        return kernels.add_layer_norm(h, w["fln.w"], w["fln.b"], cfg.eps, r1=a, r2=f)

    def forward_suffix(self, inputs_embeds, prefix_cache, key_valid=None):
        """Prefill of B prompt suffixes behind one shared prefix whose K / V rows of every layer are in `prefix_cache` (a
        generate.PagedKVCache of one sequence and one page, filled by `forward(..., cache=...)`, whose `length` is the
        prefix length P).  inputs_embeds [B,Ts,C] are positions P..P+Ts-1; key_valid [B,Ts] (True/1 = real token) or None ->
        last_hidden_state [B,Ts,C], the rows the unsplit prompts would give at those positions."""
        cfg, w = self.cfg, self.w
        B, T, C = inputs_embeds.shape
        nh, hd = cfg.heads, cfg.head_dim
        rd = int(hd * cfg.rotary_frac)
        P = prefix_cache.length
        key = ("suffix", P, T)
        if key not in self._rope:    # rotary tables of positions P..P+Ts-1 (the kernel takes tables of any length)
            cos, sin = self.rope_tables(P + T)
            self._rope[key] = (cos[P:].contiguous(), sin[P:].contiguous())
        cos, sin = self._rope[key]
        kv = None
        if key_valid is not None:
            kv = key_valid.to(device=self.device, dtype=torch.uint8).contiguous()
        h = inputs_embeds.contiguous()
        a = f = None
        for i in range(cfg.layers):
            if a is None:
                x = kernels.add_layer_norm(h, w["%d.ln.w" % i], w["%d.ln.b" % i], cfg.eps)
            else:
                h, x = kernels.add_layer_norm(h, w["%d.ln.w" % i], w["%d.ln.b" % i], cfg.eps, r1=a, r2=f, return_sum=True)
            qkv = F.linear(x, w["%d.qkv.w" % i], w["%d.qkv.b" % i]).view(B, T, 3, nh, hd)
            kernels.rotary_inplace(qkv, cos, sin, B, T, nh, hd, rd)
            # prefix pages: [1 page, nh, page_size, hd] -> head-major [nh, page_size, hd]
            a = kernels.timed("prefix_causal_attention", kernels.prefix_causal_attention, qkv, prefix_cache.k[i][0],
                              prefix_cache.v[i][0], P, kv, B, T, nh, hd)
            a = F.linear(a, w["%d.dense.w" % i], w["%d.dense.b" % i])
            f = self._fc1_gelu(x, i)
            f = F.linear(f, w["%d.fc2.w" % i], w["%d.fc2.b" % i])
        return kernels.add_layer_norm(h, w["fln.w"], w["fln.b"], cfg.eps, r1=a, r2=f)

    def decode_step(self, x, cache):
        """One autoregressive step: x [B,1,C] = embedding of the newest token of every sequence, position cache.length
        (all sequences have the same length).  Appends its K / V to the cache and returns the final hidden state [B,1,C].
        (PhiDecoderLayer with past_key_values, single-token branch of llava_phi.py:773-778.)"""
        cfg, w = self.cfg, self.w
        B, T, C = x.shape
        nh, hd = cfg.heads, cfg.head_dim
        rd = int(hd * cfg.rotary_frac)
        pos = cache.length
        cos, sin = self.rope_tables(cache.max_len)
        cos, sin = cos[pos:pos + 1].contiguous(), sin[pos:pos + 1].contiguous()
        h = x.contiguous()
        a = f = None
        for i in range(cfg.layers):
            if a is None:
                y = kernels.add_layer_norm(h, w["%d.ln.w" % i], w["%d.ln.b" % i], cfg.eps)
            else:
                h, y = kernels.add_layer_norm(h, w["%d.ln.w" % i], w["%d.ln.b" % i], cfg.eps, r1=a, r2=f, return_sum=True)
            qkv = F.linear(y, w["%d.qkv.w" % i], w["%d.qkv.b" % i]).view(B, 1, 3, nh, hd)
            kernels.rotary_inplace(qkv, cos, sin, B, 1, nh, hd, rd)
            kernels.kv_cache_write(qkv, cache.k[i], cache.v[i], cache.block_table, cache.seq_lens)
            a = kernels.paged_decode_attention(qkv, cache.k[i], cache.v[i], cache.block_table, cache.seq_lens_plus1)
            a = F.linear(a, w["%d.dense.w" % i], w["%d.dense.b" % i])
            f = F.linear(self._fc1_gelu(y, i), w["%d.fc2.w" % i], w["%d.fc2.b" % i])
        return kernels.add_layer_norm(h, w["fln.w"], w["fln.b"], cfg.eps, r1=a, r2=f)

    def _fc1_gelu(self, x, i):
        """fc1 + gelu_new: bias and tanh-GELU run in the library GEMM's epilogue (cuBLASLt) on the GPU."""
        return kernels.linear_act(x, self.w["%d.fc1.w" % i], self.w["%d.fc1.b" % i], "gelu_tanh")
