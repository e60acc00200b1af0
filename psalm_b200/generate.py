"""Chat / decoding path (SURVEY.md section 8 f4): `PSALM.generate` - prefill + greedy / sampled autoregressive decode
with a paged KV cache and the `lm_head` projection.

Restates what the reference gets from transformers' GenerationMixin on `PSALM(PhiForCausalLM, ...)` as used by
psalm/serve/cli.py:89-96 (`model.generate(input_ids, images=..., do_sample, temperature, max_new_tokens, use_cache=True)`):
the prompt may contain ONE <image> sentinel (-200), replaced by the projected image tokens (llava_arch.py:98-179); new
tokens are embedded, run through the 24 decoder layers one token at a time (single-token branch, llava_phi.py:773-778),
and `lm_head` (no bias in the reference, llava_phi.py:191) gives the next-token logits.  HF's cache grows by torch.cat
(a full copy per layer per token); here K / V live in fixed pages addressed through a block table (csrc/decode.cu)."""
import torch
import torch.nn.functional as F

from . import sequence as SEQ


class PagedKVCache:
    """Pages [num_pages, nh, page_size, hd] per layer for K and V; block_table [B, max_pages] int32.  Pages of different
    sequences are interleaved on purpose (page j of sequence b is physical page j * B + b): nothing relies on contiguity."""

    def __init__(self, phi_cfg, batch, max_len, dtype, device, page_size=16):
        self.page_size, self.max_len = page_size, int(max_len)
        self.max_pages = -(-self.max_len // page_size)
        nh, hd = phi_cfg.heads, phi_cfg.head_dim
        shape = (batch * self.max_pages, nh, page_size, hd)
        self.k = [torch.empty(shape, dtype=dtype, device=device) for _ in range(phi_cfg.layers)]
        self.v = [torch.empty(shape, dtype=dtype, device=device) for _ in range(phi_cfg.layers)]
        # built on the device (no host copy), so that a cache can also be allocated inside a CUDA graph capture
        bt = torch.arange(self.max_pages * batch, dtype=torch.int32, device=device).view(self.max_pages, batch)
        self.block_table = bt.t().contiguous()
        self.length = 0
        self.seq_lens = torch.zeros(batch, dtype=torch.int32, device=device)          # tokens already cached
        self.seq_lens_plus1 = torch.ones(batch, dtype=torch.int32, device=device)     # ... including the one being decoded

    def advance(self, n):
        self.length += n
        if self.length > self.max_len:
            raise RuntimeError("PagedKVCache: %d tokens exceed the allocated %d" % (self.length, self.max_len))
        self.seq_lens.fill_(self.length)
        self.seq_lens_plus1.fill_(self.length + 1)


def chat_embeds(model, input_ids, images=None):
    """input_ids [B,T0] with at most one <image> sentinel per row -> inputs_embeds [B,T,C] (equal lengths required)."""
    ids = input_ids.to(model.device)
    emb = model.model.embed_tokens
    img_tok = None
    if images is not None:
        img_tok = model.encode_images(images.to(model.device))
    rows = []
    for b in range(ids.shape[0]):
        row = ids[b]
        pos = (row == SEQ.IMAGE_TOKEN_INDEX).nonzero().flatten().tolist()
        if (row < 0).sum().item() != len(pos):
            raise NotImplementedError("generate(): only the <image> sentinel is valid in a chat prompt")
        if len(pos) > 1:
            raise AssertionError("not supporting multi image index")          # llava_phi.py:588
        if pos:
            if img_tok is None:
                raise ValueError("the prompt has an <image> token but no image was given")
            p = pos[0]
            rows.append(torch.cat([emb[row[:p]], img_tok[b].to(emb.dtype), emb[row[p + 1:]]], 0))
        else:
            rows.append(emb[row])
    if len({r.shape[0] for r in rows}) != 1:
        raise NotImplementedError("generate(): prompts of one batch must have the same length (serve one request per call)")
    return torch.stack(rows, 0).contiguous()


@torch.no_grad()
def generate(model, input_ids, images=None, max_new_tokens=32, do_sample=False, temperature=1.0, top_p=None,
             eos_token_id=None, generator=None, page_size=16):
    """Returns the generated token ids [B, n_new] (the prompt is not repeated)."""
    if model.lm_head is None:
        raise RuntimeError("generate(): the checkpoint has no lm_head.weight")
    with model._precision_scope():
        embeds = chat_embeds(model, input_ids, images)
        B, T, _ = embeds.shape
        phi = model.model.phi
        cache = PagedKVCache(phi.cfg, B, T + max_new_tokens, model.dtype, model.device, page_size)
        hidden = phi.forward(embeds, None, cache=cache)
        cache.advance(T)
        last = hidden[:, -1]
        out = []
        done = torch.zeros(B, dtype=torch.bool, device=model.device)
        for step in range(max_new_tokens):
            logits = F.linear(last, model.lm_head[0], model.lm_head[1]).float()
            if do_sample:
                probs = torch.softmax(logits / max(float(temperature), 1e-5), -1)
                if top_p is not None and top_p < 1.0:
                    sp, si = torch.sort(probs, -1, descending=True)
                    keep = (sp.cumsum(-1) - sp) < top_p
                    sp = sp * keep
                    probs = torch.zeros_like(probs).scatter_(-1, si, sp / sp.sum(-1, keepdim=True))
                tok = torch.multinomial(probs, 1, generator=generator).squeeze(-1)
            else:
                tok = logits.argmax(-1)
            out.append(tok)
            if eos_token_id is not None:
                done |= tok == eos_token_id
                if bool(done.all()):
                    break
            if step + 1 == max_new_tokens:
                break
            x = model.model.embed_tokens[tok].unsqueeze(1)
            last = phi.decode_step(x, cache)[:, 0]
            cache.advance(1)
        return torch.stack(out, 1)
