"""TEST INFRASTRUCTURE — CPU restatement (plain PyTorch fp32/fp64, functional, no custom kernels) of
the reference `PSALM.eval_seg` path.  Only tests/, `__graft_entry__.smoke()` and bench.py's
cpu_baseline / `--impl reference` legs may import this module; nothing under psalm_b200/ does.

Every function cites the reference lines it restates.  Abbreviations (relative to
psalm/model/ of the reference):
  LP   = language_model/llava_phi.py
  SWIN = multimodal_encoder/swin_trans.py
  PROJ = multimodal_projector/builder.py
  PIX  = mask_decoder/Mask2Former_Simplify/modeling/pixel_decoder/msdeformattn.py
  OPS  = mask_decoder/Mask2Former_Simplify/modeling/pixel_decoder/ops/
  DEC  = mask_decoder/Mask2Former_Simplify/modeling/transformer_decoder/mask2former_transformer_decoder.py
  POS  = mask_decoder/Mask2Former_Simplify/modeling/transformer_decoder/position_encoding.py
  PHI  = transformers/models/phi/modeling_phi.py  (third-party; reference pins transformers==4.36.2,
         pyproject.toml:27; restated from the installed 5.5.0 eager path — same mathematics)

Pinning: oracle/gen_golden.py runs the *unmodified reference modules* (through oracle/ref_shims.py)
and this restatement on the same weights/inputs and commits the reference outputs to tests/golden/;
tests/test_oracle_golden.py re-checks this file against those fixtures everywhere (no reference
needed).  Third-party arithmetic with no reference-side test (PHI, detectron2 post-processing) is
"parity unpinned" upstream; here it is pinned only to what the reference produced in this container.

State dict `sd`: the reference checkpoint layout (SURVEY.md Appendix B), tensors on CPU.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

IMAGE_TOKEN_INDEX = -200   # psalm/constants.py:8-12
SEG_TOKEN_INDEX = -201
CLS_TOKEN_INDEX = -202
REGION_TOKEN_INDEX = -203
REFER_TOKEN_INDEX = -204


def _lin(sd, name, x):
    return F.linear(x, sd[name + ".weight"], sd.get(name + ".bias"))


def _ln(sd, name, x, eps=1e-5):
    return F.layer_norm(x, (x.shape[-1],), sd[name + ".weight"], sd[name + ".bias"], eps)


# ------------------------------------------------------------------------------------------------
# MSDeformAttn core — OPS/functions/ms_deform_attn_func.py:52-78 (ms_deform_attn_core_pytorch)
# ------------------------------------------------------------------------------------------------
def msda_core(value, spatial_shapes, sampling_locations, attention_weights):
    """value [N,S,M,D]; spatial_shapes list[(H,W)]; loc [N,Lq,M,L,P,2]; w [N,Lq,M,L,P] -> [N,Lq,M*D]."""
    N, S, M, D = value.shape
    _, Lq, _, L, P, _ = sampling_locations.shape
    shapes = [(int(h), int(w)) for h, w in spatial_shapes]
    value_list = value.split([h * w for h, w in shapes], dim=1)
    grids = 2 * sampling_locations - 1
    sampled = []
    for lid, (H, W) in enumerate(shapes):
        v = value_list[lid].flatten(2).transpose(1, 2).reshape(N * M, D, H, W)
        g = grids[:, :, :, lid].transpose(1, 2).flatten(0, 1)
        sampled.append(F.grid_sample(v, g, mode="bilinear", padding_mode="zeros", align_corners=False))
    aw = attention_weights.transpose(1, 2).reshape(N * M, 1, Lq, L * P)
    out = (torch.stack(sampled, dim=-2).flatten(-2) * aw).sum(-1).view(N, M * D, Lq)
    return out.transpose(1, 2).contiguous()


# ------------------------------------------------------------------------------------------------
# Sine position embedding — POS:29-52 (normalize=True, scale=2*pi, T=1e4, num_pos_feats=128)
# ------------------------------------------------------------------------------------------------
def position_embedding_sine(B, H, W, num_pos_feats=128, temperature=10000.0):
    not_mask = torch.ones(B, H, W, dtype=torch.bool)
    y_embed = not_mask.cumsum(1, dtype=torch.float32)
    x_embed = not_mask.cumsum(2, dtype=torch.float32)
    eps, scale = 1e-6, 2 * math.pi
    y_embed = y_embed / (y_embed[:, -1:, :] + eps) * scale
    x_embed = x_embed / (x_embed[:, :, -1:] + eps) * scale
    dim_t = torch.arange(num_pos_feats, dtype=torch.float32)
    dim_t = temperature ** (2 * torch.div(dim_t, 2, rounding_mode="floor") / num_pos_feats)
    pos_x = x_embed[:, :, :, None] / dim_t
    pos_y = y_embed[:, :, :, None] / dim_t
    pos_x = torch.stack((pos_x[:, :, :, 0::2].sin(), pos_x[:, :, :, 1::2].cos()), dim=4).flatten(3)
    pos_y = torch.stack((pos_y[:, :, :, 0::2].sin(), pos_y[:, :, :, 1::2].cos()), dim=4).flatten(3)
    return torch.cat((pos_y, pos_x), dim=3).permute(0, 3, 1, 2)  # [B,256,H,W]


# ------------------------------------------------------------------------------------------------
# Swin — SWIN:608-633 and callees
# ------------------------------------------------------------------------------------------------
SWIN_B = dict(embed_dim=128, depths=(2, 2, 18, 2), num_heads=(4, 8, 16, 32), window=12)  # SWIN:660-678


def _window_partition(x, ws):  # SWIN:36-48
    B, H, W, C = x.shape
    x = x.view(B, H // ws, ws, W // ws, ws, C)
    return x.permute(0, 1, 3, 2, 4, 5).contiguous().view(-1, ws, ws, C)


def _window_reverse(windows, ws, H, W):  # SWIN:51-65
    B = int(windows.shape[0] / (H * W / ws / ws))
    x = windows.view(B, H // ws, W // ws, ws, ws, -1)
    return x.permute(0, 1, 3, 2, 4, 5).contiguous().view(B, H, W, -1)


def relative_position_index(ws):  # SWIN:93-103
    coords = torch.stack(torch.meshgrid([torch.arange(ws), torch.arange(ws)], indexing="ij"))
    cf = torch.flatten(coords, 1)
    rel = (cf[:, :, None] - cf[:, None, :]).permute(1, 2, 0).contiguous()
    rel[:, :, 0] += ws - 1
    rel[:, :, 1] += ws - 1
    rel[:, :, 0] *= 2 * ws - 1
    return rel.sum(-1)


def _window_attention(sd, pre, x, mask, nh, ws):  # SWIN:117-149
    B_, N, C = x.shape
    qkv = _lin(sd, pre + "qkv", x).reshape(B_, N, 3, nh, C // nh).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0], qkv[1], qkv[2]
    q = q * ((C // nh) ** -0.5)
    attn = q @ k.transpose(-2, -1)
    idx = sd.get(pre + "relative_position_index")
    if idx is None:
        idx = relative_position_index(ws)
    bias = sd[pre + "relative_position_bias_table"][idx.view(-1)].view(N, N, -1).permute(2, 0, 1).contiguous()
    attn = attn + bias.unsqueeze(0)
    if mask is not None:
        nW = mask.shape[0]
        attn = attn.view(B_ // nW, nW, nh, N, N) + mask.unsqueeze(1).unsqueeze(0)
        attn = attn.view(-1, nh, N, N)
    attn = attn.softmax(dim=-1)
    x = (attn @ v).transpose(1, 2).reshape(B_, N, C)
    return _lin(sd, pre + "proj", x)


def _swin_block(sd, pre, x, H, W, nh, ws, shift, mask_matrix):  # SWIN:194-253
    B, L, C = x.shape
    shortcut = x
    x = _ln(sd, pre + "norm1", x).view(B, H, W, C)
    pad_r = (ws - W % ws) % ws
    pad_b = (ws - H % ws) % ws
    x = F.pad(x, (0, 0, 0, pad_r, 0, pad_b))  # zeros AFTER norm1 (SWIN:207-214)
    _, Hp, Wp, _ = x.shape
    if shift > 0:
        shifted = torch.roll(x, shifts=(-shift, -shift), dims=(1, 2))
        attn_mask = mask_matrix
    else:
        shifted, attn_mask = x, None
    xw = _window_partition(shifted, ws).view(-1, ws * ws, C)
    aw = _window_attention(sd, pre + "attn.", xw, attn_mask, nh, ws).view(-1, ws, ws, C)
    shifted = _window_reverse(aw, ws, Hp, Wp)
    x = torch.roll(shifted, shifts=(shift, shift), dims=(1, 2)) if shift > 0 else shifted
    if pad_r > 0 or pad_b > 0:
        x = x[:, :H, :W, :].contiguous()
    x = shortcut + x.view(B, H * W, C)
    h = _lin(sd, pre + "mlp.fc2", F.gelu(_lin(sd, pre + "mlp.fc1", _ln(sd, pre + "norm2", x))))  # SWIN:16-34
    return x + h


def _shift_mask(H, W, ws, shift):  # SWIN:370-387
    Hp = int(np.ceil(H / ws)) * ws
    Wp = int(np.ceil(W / ws)) * ws
    img_mask = torch.zeros((1, Hp, Wp, 1))
    cnt = 0
    for h in (slice(0, -ws), slice(-ws, -shift), slice(-shift, None)):
        for w in (slice(0, -ws), slice(-ws, -shift), slice(-shift, None)):
            img_mask[:, h, w, :] = cnt
            cnt += 1
    mw = _window_partition(img_mask, ws).view(-1, ws * ws)
    am = mw.unsqueeze(1) - mw.unsqueeze(2)
    return am.masked_fill(am != 0, float(-100.0)).masked_fill(am == 0, float(0.0))


def swin_forward(sd, pre, x, cfg=SWIN_B):
    """x [B,3,H,W] -> (res2,res3,res4,res5) NCHW.  SWIN:608-633."""
    ws = cfg["window"]
    _, _, H, W = x.shape  # PatchEmbed SWIN:427-443
    if W % 4 != 0:
        x = F.pad(x, (0, 4 - W % 4))
    if H % 4 != 0:
        x = F.pad(x, (0, 0, 0, 4 - H % 4))
    x = F.conv2d(x, sd[pre + "patch_embed.proj.weight"], sd[pre + "patch_embed.proj.bias"], stride=4)
    Wh, Ww = x.shape[2], x.shape[3]
    x = _ln(sd, pre + "patch_embed.norm", x.flatten(2).transpose(1, 2))
    outs = []
    for i, depth in enumerate(cfg["depths"]):
        nh = cfg["num_heads"][i]
        mask = _shift_mask(Wh, Ww, ws, ws // 2)
        for j in range(depth):
            x = _swin_block(sd, "%slayers.%d.blocks.%d." % (pre, i, j), x, Wh, Ww, nh, ws,
                            0 if j % 2 == 0 else ws // 2, mask)
        C = x.shape[-1]
        out = _ln(sd, "%snorm%d" % (pre, i), x)
        outs.append(out.view(-1, Wh, Ww, C).permute(0, 3, 1, 2).contiguous())
        if i < len(cfg["depths"]) - 1:  # PatchMerging SWIN:269-296
            B = x.shape[0]
            xm = x.view(B, Wh, Ww, C)
            if Wh % 2 == 1 or Ww % 2 == 1:
                xm = F.pad(xm, (0, 0, 0, Ww % 2, 0, Wh % 2))
            xm = torch.cat([xm[:, 0::2, 0::2], xm[:, 1::2, 0::2], xm[:, 0::2, 1::2], xm[:, 1::2, 1::2]], -1)
            xm = xm.view(B, -1, 4 * C)
            x = F.linear(_ln(sd, "%slayers.%d.downsample.norm" % (pre, i), xm),
                         sd["%slayers.%d.downsample.reduction.weight" % (pre, i)])
            Wh, Ww = (Wh + 1) // 2, (Ww + 1) // 2
    return tuple(outs)


# ------------------------------------------------------------------------------------------------
# Projector — PROJ:365-375 (ResNetSwin) / PROJ:85-111 (BasicBlock, conv2 applied TWICE at :92-94)
# ------------------------------------------------------------------------------------------------
def _bn(sd, name, x, eps=1e-5):
    return F.batch_norm(x, sd[name + ".running_mean"], sd[name + ".running_var"], sd[name + ".weight"],
                        sd[name + ".bias"], False, 0.0, eps)


def projector_forward(sd, pre, res5):
    b = pre + "layer1.0."
    out = F.relu(_bn(sd, b + "bn1", F.conv2d(res5, sd[b + "conv1.weight"], None, stride=2, padding=1)))
    out = F.conv2d(out, sd[b + "conv2.weight"], None, padding=1)
    out = F.conv2d(out, sd[b + "conv2.weight"], None, padding=1)
    out = _bn(sd, b + "bn2", out)
    res = _bn(sd, b + "downsample.1", F.conv2d(res5, sd[b + "downsample.0.weight"], None, stride=2))
    out = F.relu(out + res)
    out = out.reshape(out.shape[0], out.shape[1], -1).permute(0, 2, 1)
    return _lin(sd, pre + "fc", out)


# ------------------------------------------------------------------------------------------------
# Region prompts — visual_prompt_module/context_cluster.py:31-40 (rand_sample_repeat), :43-68 (point_sample),
# :333-400 (region_pooling); called from LP:791-797
# ------------------------------------------------------------------------------------------------
def sample_region_points(region_masks, num_sample_point=256):
    """region_masks [K,H,W] (bool / 0-1) -> [K, num_sample_point, 2] normalised (y / H, x / W) positions of mask
    pixels.  Draws from the GLOBAL CPU generator with the reference's calls in the reference's order (torch.randint
    when a mask has fewer pixels than points, torch.randperm when it has more, context_cluster.py:31-40), so the
    same torch.manual_seed gives the same points as the reference."""
    wh = torch.tensor([region_masks[0].shape[0], region_masks[0].shape[1]])[None]
    out = []
    for m in region_masks:
        x = m.nonzero() / wh
        if x.shape[0] < num_sample_point:
            idx = torch.randint(0, x.shape[0], (num_sample_point - x.shape[0],))
            x = torch.cat((x, x[idx]), dim=0)
        elif x.shape[0] > num_sample_point:
            x = x[torch.randperm(x.shape[0])[:num_sample_point], :]
        out.append(x)
    return torch.stack(out)


def region_pool(img_tok_b, points):
    """img_tok_b [n_img, C] (projector output of one image, h = w = sqrt(n_img)); points [K,P,2] (y, x) in [0,1]
    -> [K, 1, C]: grid_sample(align_corners=True) at the points, mean over P (context_cluster.py:355-371, :392)."""
    h = w = int(math.sqrt(img_tok_b.shape[0]))
    c = img_tok_b.shape[-1]
    fmap = img_tok_b.reshape(h, w, c).permute(2, 0, 1).unsqueeze(0).repeat(points.shape[0], 1, 1, 1)
    grid = (2.0 * points.flip(dims=(2,)).to(img_tok_b.dtype) - 1.0).unsqueeze(2)
    fea = F.grid_sample(fmap.float(), grid.float(), align_corners=True).squeeze(3).to(img_tok_b.dtype)   # [K,C,P]
    return fea.mean(-1).unsqueeze(1)


# ------------------------------------------------------------------------------------------------
# Sequence assembly — LP:767-971 / LP:581-766 (batch of B samples, ragged -> right padded)
# ------------------------------------------------------------------------------------------------
def assemble_sequence(sd, input_ids, attention_mask, image_features, class_name_ids=None, cls_indices=None,
                      class_name_embedding_indices=None, token_refer_id=None, refer_embedding_indices=None,
                      region_features=None):
    """Returns dict(inputs_embeds [B,T,C], attention_mask [B,T] bool, seg_query_mask [B,T],
    class_name_embedding_indices [B,T] or None, refer_embedding_indices [B,T] or None, region_embedding_masks [B,T] or
    None).  region_features: per sample [K,1,C] (LP:795-797), one per <region> token in order (LP:685-703)."""
    emb = sd["model.embed_tokens.weight"]
    seg_query = sd["seg_query"]
    B = input_ids.shape[0]
    per = []
    for b in range(B):
        ids = input_ids[b]
        # embed_class_ids LP:566-575
        cls_embeds = None
        if class_name_ids is not None:
            ci = cls_indices[b]
            uniq = ci.unique_consecutive()
            uniq = uniq[uniq >= 0]
            cls_embeds = [emb[class_name_ids[b][ci == u]] for u in uniq]
        refer_embed = emb[token_refer_id[b]] if token_refer_id is not None else None  # LP:576-580
        embeds, qmask, cidx, ridx, gmask = [], [], [], [], []
        cls_i = 0
        region_i = 0
        if region_features is not None:
            assert (ids == REGION_TOKEN_INDEX).sum() == len(region_features[b])  # LP:592-594
        assert (ids == IMAGE_TOKEN_INDEX).sum() == 1 and (ids == SEG_TOKEN_INDEX).sum() == 1  # LP:588-589
        if cls_embeds is not None:
            assert (ids == CLS_TOKEN_INDEX).sum() == len(cls_embeds)  # LP:590-591
        i = 0
        n = ids.shape[0]
        while i < n:  # chunking LP:614-746
            t = int(ids[i])
            if t >= 0:
                j = i
                while j < n and int(ids[j]) >= 0:
                    j += 1
                embeds.append(emb[ids[i:j]])
                k = j - i
                qmask.append(torch.zeros(k))
                cidx.append(class_name_embedding_indices[b][i:j] if class_name_embedding_indices is not None
                            else torch.zeros(k, dtype=torch.long))
                ridx.append(refer_embedding_indices[b][i:j] if refer_embedding_indices is not None
                            else torch.zeros(k, dtype=torch.long))
                gmask.append(torch.zeros(k))
                i = j
                continue
            if t == IMAGE_TOKEN_INDEX:
                e, qm, cv, rv = image_features[b], 0, 0, 0
            elif t == SEG_TOKEN_INDEX:
                e, qm, cv, rv = seg_query, 1, 0, 0
            elif t == CLS_TOKEN_INDEX:
                e = cls_embeds[cls_i]
                cls_i += 1
                qm, cv, rv = 0, cls_i, 0  # index value = running 1-based class counter (LP:671-673)
            elif t == REFER_TOKEN_INDEX:
                e, qm, cv, rv = refer_embed, 0, 0, 1
            elif t == REGION_TOKEN_INDEX:   # LP:684-703
                e, qm, cv, rv = region_features[b][region_i], 0, 0, 0
                region_i += 1
            else:
                raise ValueError("unknown sentinel id %d" % t)
            if e.dim() == 1:
                e = e.unsqueeze(0)
            k = e.shape[0]
            gmask.append(torch.full((k,), 1.0 if t == REGION_TOKEN_INDEX else 0.0))
            embeds.append(e)
            qmask.append(torch.full((k,), float(qm)))
            cidx.append(torch.full((k,), cv, dtype=torch.long))
            ridx.append(torch.full((k,), rv, dtype=torch.long))
            i += 1
        per.append((torch.cat(embeds, 0), torch.cat(qmask, 0), torch.cat(cidx, 0), torch.cat(ridx, 0), torch.cat(gmask, 0)))
    T = max(p[0].shape[0] for p in per)
    C = per[0][0].shape[1]
    out_e = torch.zeros(B, T, C, dtype=per[0][0].dtype)
    out_q = torch.zeros(B, T)
    out_c = torch.zeros(B, T, dtype=torch.long)
    out_r = torch.zeros(B, T, dtype=torch.long)
    out_m = torch.zeros(B, T, dtype=torch.bool)
    out_g = torch.zeros(B, T)
    for b, (e, qm, cv, rv, gm) in enumerate(per):
        t = e.shape[0]
        out_e[b, :t], out_q[b, :t], out_c[b, :t], out_r[b, :t], out_g[b, :t] = e, qm, cv, rv, gm
        # LP:935-949 / 964-969: new tokens are attendable, then the caller's mask, then right padding False
        left = t - input_ids.shape[1]
        out_m[b, :left] = True
        out_m[b, left:t] = attention_mask[b].bool()
    return dict(inputs_embeds=out_e, attention_mask=out_m, seg_query_mask=out_q,
                class_name_embedding_indices=out_c if class_name_embedding_indices is not None else None,
                refer_embedding_indices=out_r if refer_embedding_indices is not None else None,
                region_embedding_masks=out_g if region_features is not None else None)


# ------------------------------------------------------------------------------------------------
# Phi — PHI (PhiModel.forward, PhiDecoderLayer, PhiAttention eager, PhiMLP gelu_new)
# ------------------------------------------------------------------------------------------------
PHI_15 = dict(hidden=2048, layers=24, heads=32, inter=8192, eps=1e-5, theta=10000.0, rotary_frac=0.5)


def gelu_new(x):
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * torch.pow(x, 3.0))))


def phi_forward(sd, pre, inputs_embeds, attention_mask, cfg=PHI_15):
    """inputs_embeds [B,T,C]; attention_mask [B,T] bool (True = real token) -> last_hidden_state."""
    B, T, C = inputs_embeds.shape
    nh = cfg["heads"]
    hd = C // nh
    rd = int(hd * cfg["rotary_frac"])
    inv_freq = 1.0 / (cfg["theta"] ** (torch.arange(0, rd, 2, dtype=torch.int64).float() / rd))
    freqs = torch.arange(T).float()[:, None] * inv_freq[None, :]
    emb = torch.cat((freqs, freqs), dim=-1)
    cos, sin = emb.cos()[None, None], emb.sin()[None, None]
    neg = torch.finfo(inputs_embeds.dtype).min
    causal = torch.tril(torch.ones(T, T, dtype=torch.bool))
    allowed = causal[None, None] & attention_mask[:, None, None, :].bool()
    bias = torch.zeros(B, 1, T, T, dtype=inputs_embeds.dtype).masked_fill(~allowed, neg)

    def rot_half(x):
        x1, x2 = x[..., : x.shape[-1] // 2], x[..., x.shape[-1] // 2:]
        return torch.cat((-x2, x1), dim=-1)

    h = inputs_embeds
    for i in range(cfg["layers"]):
        p = "%slayers.%d." % (pre, i)
        res = h
        x = _ln(sd, p + "input_layernorm", h, cfg["eps"])
        q = _lin(sd, p + "self_attn.q_proj", x).view(B, T, nh, hd).transpose(1, 2)
        k = _lin(sd, p + "self_attn.k_proj", x).view(B, T, nh, hd).transpose(1, 2)
        v = _lin(sd, p + "self_attn.v_proj", x).view(B, T, nh, hd).transpose(1, 2)
        qr, qp = q[..., :rd], q[..., rd:]
        kr, kp = k[..., :rd], k[..., rd:]
        qr = qr * cos + rot_half(qr) * sin
        kr = kr * cos + rot_half(kr) * sin
        q = torch.cat((qr, qp), -1)
        k = torch.cat((kr, kp), -1)
        aw = torch.matmul(q, k.transpose(2, 3)) * (hd ** -0.5) + bias
        aw = F.softmax(aw, dim=-1, dtype=torch.float32).to(q.dtype)
        ao = torch.matmul(aw, v).transpose(1, 2).reshape(B, T, C)
        ao = _lin(sd, p + "self_attn.dense", ao)
        ff = _lin(sd, p + "mlp.fc2", gelu_new(_lin(sd, p + "mlp.fc1", x)))
        h = ao + ff + res
    return _ln(sd, pre + "final_layernorm", h, cfg["eps"])


# ------------------------------------------------------------------------------------------------
# Pixel decoder — PIX:268-315, encoder PIX:136-164 / 89-95 / 57-66, MSDeformAttn OPS/modules/ms_deform_attn.py:82-124
# ------------------------------------------------------------------------------------------------
def _gn(sd, name, x, groups=32):
    return F.group_norm(x, groups, sd[name + ".weight"], sd[name + ".bias"], 1e-5)


def msdeform_attn_module(sd, pre, query, reference_points, src, shapes, n_heads=8, n_points=4):
    N, Lq, C = query.shape
    L = len(shapes)
    value = _lin(sd, pre + "value_proj", src).view(N, src.shape[1], n_heads, C // n_heads)
    off = _lin(sd, pre + "sampling_offsets", query).view(N, Lq, n_heads, L, n_points, 2)
    aw = _lin(sd, pre + "attention_weights", query).view(N, Lq, n_heads, L * n_points)
    aw = F.softmax(aw, -1).view(N, Lq, n_heads, L, n_points)
    normalizer = torch.tensor([[w, h] for h, w in shapes], dtype=query.dtype)
    loc = reference_points[:, :, None, :, None, :] + off / normalizer[None, None, None, :, None, :]
    out = msda_core(value, shapes, loc, aw)
    return _lin(sd, pre + "output_proj", out)


def encoder_reference_points(shapes, B):  # PIX:76-87 with valid_ratios == 1
    refs = []
    for H, W in shapes:
        ry, rx = torch.meshgrid(torch.linspace(0.5, H - 0.5, H), torch.linspace(0.5, W - 0.5, W), indexing="ij")
        refs.append(torch.stack((rx.reshape(-1)[None] / W, ry.reshape(-1)[None] / H), -1))
    ref = torch.cat(refs, 1)  # [1,S,2]
    return ref[:, :, None].expand(B, -1, len(shapes), -1)


def pixel_decoder_forward(sd, pre, feats):
    """feats dict res2..res5 NCHW -> (mask_features, enc_res5_level, [3 multi-scale maps])."""
    srcs, poss = [], []
    for idx, f in enumerate(("res5", "res4", "res3")):  # PIX:272-276
        x = feats[f]
        p = "%sinput_proj.%d." % (pre, idx)
        srcs.append(_gn(sd, p + "1", F.conv2d(x, sd[p + "0.weight"], sd[p + "0.bias"])))
        poss.append(position_embedding_sine(x.shape[0], x.shape[2], x.shape[3]).to(x.dtype))
    B = srcs[0].shape[0]
    shapes = [(s.shape[2], s.shape[3]) for s in srcs]
    src = torch.cat([s.flatten(2).transpose(1, 2) for s in srcs], 1)
    level_embed = sd[pre + "transformer.level_embed"]
    pos = torch.cat([p.flatten(2).transpose(1, 2) + level_embed[l].view(1, 1, -1) for l, p in enumerate(poss)], 1)
    ref = encoder_reference_points(shapes, B)
    out = src
    n_layers = 0
    while "%stransformer.encoder.layers.%d.norm1.weight" % (pre, n_layers) in sd:
        n_layers += 1
    for i in range(n_layers):  # PIX:57-66
        p = "%stransformer.encoder.layers.%d." % (pre, i)
        s2 = msdeform_attn_module(sd, p + "self_attn.", out + pos, ref, out, shapes)
        out = _ln(sd, p + "norm1", out + s2)
        s2 = _lin(sd, p + "linear2", F.relu(_lin(sd, p + "linear1", out)))
        out = _ln(sd, p + "norm2", out + s2)
    ys = torch.split(out, [h * w for h, w in shapes], dim=1)
    outs = [z.transpose(1, 2).reshape(B, -1, h, w) for z, (h, w) in zip(ys, shapes)]
    x = feats["res2"]  # FPN level PIX:300-309
    cur = F.relu(_gn(sd, pre + "adapter_1.1", F.conv2d(x, sd[pre + "adapter_1.0.weight"], sd[pre + "adapter_1.0.bias"])))
    y = cur + F.interpolate(outs[-1].float(), size=cur.shape[-2:], mode="bilinear", align_corners=False).to(x.dtype)
    y = F.relu(_gn(sd, pre + "layer_1.1", F.conv2d(y, sd[pre + "layer_1.0.weight"], sd[pre + "layer_1.0.bias"], padding=1)))
    outs.append(y)
    mask_features = F.conv2d(outs[-1], sd[pre + "mask_features.weight"], sd[pre + "mask_features.bias"])
    return mask_features, outs[0], outs[:3]


# ------------------------------------------------------------------------------------------------
# Masked-attention decoder — DEC:596-693 (forward_woconcat), DEC:695-762 (prediction heads)
# ------------------------------------------------------------------------------------------------
def _mha(sd, pre, q, k, v, nh, attn_mask=None):
    """nn.MultiheadAttention forward (seq-first), packed in_proj (DEC:18,75)."""
    Lq, B, C = q.shape
    Lk = k.shape[0]
    W, bias = sd[pre + "in_proj_weight"], sd[pre + "in_proj_bias"]
    hd = C // nh
    qp = F.linear(q, W[:C], bias[:C]).view(Lq, B * nh, hd).transpose(0, 1)
    kp = F.linear(k, W[C:2 * C], bias[C:2 * C]).view(Lk, B * nh, hd).transpose(0, 1)
    vp = F.linear(v, W[2 * C:], bias[2 * C:]).view(Lk, B * nh, hd).transpose(0, 1)
    qp = qp * math.sqrt(1.0 / hd)
    attn = torch.bmm(qp, kp.transpose(1, 2))
    if attn_mask is not None:
        attn = attn.masked_fill(attn_mask, float("-inf"))
    attn = F.softmax(attn, dim=-1)
    out = torch.bmm(attn, vp).transpose(0, 1).contiguous().view(Lq, B, C)
    return _lin(sd, pre + "out_proj", out)


def _mlp(sd, pre, x, n):  # DEC:187-199
    for i in range(n):
        x = _lin(sd, "%slayers.%d" % (pre, i), x)
        if i < n - 1:
            x = F.relu(x)
    return x


def prediction_heads(sd, pre, output, mask_features, target_size, SEG_embedding, class_name_embedding, nh=8,
                     region_embedding_list=None, region_out=None):
    dec = _ln(sd, pre + "decoder_norm", output).transpose(0, 1)
    if region_embedding_list is not None and region_out is not None:   # DEC:737-745 (seg_proj is on)
        dr = _mlp(sd, pre + "REGION_proj.", dec, 2)
        region_out.append([torch.einsum("kd,ld->kl", re, d) for d, re in zip(dr, region_embedding_list)])
    SEG_class = None
    if SEG_embedding is not None:
        SEG_class = torch.einsum("bld,bcd->blc", _mlp(sd, pre + "SEG_proj.", dec, 2), SEG_embedding)
    cls = None
    if class_name_embedding is not None:
        cls = torch.einsum("bld,bcd->blc", _mlp(sd, pre + "CLASS_proj.", dec, 2), class_name_embedding)
    mask_embed = _mlp(sd, pre + "mask_embed.", dec, 3)
    outputs_mask = torch.einsum("bqc,bchw->bqhw", mask_embed, mask_features)
    am = F.interpolate(outputs_mask.float(), size=target_size, mode="bilinear", align_corners=False).to(mask_embed.dtype)
    am = (am.sigmoid().flatten(2).unsqueeze(1).repeat(1, nh, 1, 1).flatten(0, 1) < 0.5).bool()
    return SEG_class, cls, outputs_mask, am


def predictor_forward(sd, pre, ms_feats, mask_features, seg_query, SEG_embedding=None, class_name_embedding=None,
                      nh=8, return_all=False, region_embedding_list=None):
    src, pos, sizes = [], [], []
    for i in range(3):  # DEC:607-614  (input_proj is identity: in_channels == hidden_dim, DEC:475-479)
        x = ms_feats[i]
        sizes.append(x.shape[-2:])
        pos.append(position_embedding_sine(x.shape[0], x.shape[2], x.shape[3]).flatten(2).to(x.dtype).permute(2, 0, 1))
        src.append((x.flatten(2) + sd[pre + "level_embed.weight"][i][None, :, None]).permute(2, 0, 1))
    bs = src[0].shape[1]
    query_embed = sd[pre + "query_embed.weight"].unsqueeze(1).repeat(1, bs, 1)  # DEC:619
    output = seg_query.permute(1, 0, 2)
    region_trace = []
    SEGc, clsc, omask, attn_mask = prediction_heads(sd, pre, output, mask_features, sizes[0], SEG_embedding,
                                                    class_name_embedding, nh, region_embedding_list, region_trace)
    trace = [(SEGc, clsc, omask, attn_mask)]
    layer_outputs = [output]        # decoder state before layer 0, then after every layer ([Q, B, C])
    n_layers = 0
    while "%stransformer_ffn_layers.%d.norm.weight" % (pre, n_layers) in sd:
        n_layers += 1
    for i in range(n_layers):
        li = i % 3
        attn_mask = attn_mask.clone()
        attn_mask[torch.where(attn_mask.sum(-1) == attn_mask.shape[-1])] = False  # DEC:647
        p = "%stransformer_cross_attention_layers.%d." % (pre, i)  # DEC:93-105
        t2 = _mha(sd, p + "multihead_attn.", output + query_embed, src[li] + pos[li], src[li], nh, attn_mask)
        output = _ln(sd, p + "norm", output + t2)
        p = "%stransformer_self_attention_layers.%d." % (pre, i)  # DEC:35-45
        qk = output + query_embed
        t2 = _mha(sd, p + "self_attn.", qk, qk, output, nh)
        output = _ln(sd, p + "norm", output + t2)
        p = "%stransformer_ffn_layers.%d." % (pre, i)  # DEC:158-162
        t2 = _lin(sd, p + "linear2", F.relu(_lin(sd, p + "linear1", output)))
        output = _ln(sd, p + "norm", output + t2)
        SEGc, clsc, omask, attn_mask = prediction_heads(sd, pre, output, mask_features, sizes[(i + 1) % 3],
                                                        SEG_embedding, class_name_embedding, nh, region_embedding_list,
                                                        region_trace)
        trace.append((SEGc, clsc, omask, attn_mask))
        layer_outputs.append(output)
    out = dict(pred_SEG_logits=SEGc, pred_class_name_logits=clsc, pred_masks=omask,
               pred_region_logits=region_trace[-1] if region_trace else None)
    if return_all:
        out["trace"] = trace
        out["layer_outputs"] = layer_outputs
    return out


# ------------------------------------------------------------------------------------------------
# Embedding extraction — LP:1299-1316, LP:552-565, LP:972-978
# ------------------------------------------------------------------------------------------------
def get_seg_query(hidden, seg_query_mask):
    return torch.stack([h[m == 1] for h, m in zip(hidden, seg_query_mask) if m.sum() > 0], 0)


def get_class_name_embedding(hidden, cls_idx):
    outs = []
    for h, ci in zip(hidden, cls_idx):
        ids = torch.unique(ci)
        ids = ids[ids != 0]
        outs.append(torch.stack([h[ci == i].mean(0) for i in ids], 0))  # AdaptiveAvgPool1d(1) == mean
    return torch.stack(outs, 0)


def get_SEG_embedding(hidden, refer_idx):
    return torch.stack([h[r.bool()].mean(0, keepdim=True) for h, r in zip(hidden, refer_idx)], 0)


# ------------------------------------------------------------------------------------------------
# Post-processing — LP:1395-1472 and LP:308-447; detectron2 pieces restated (unpinned upstream)
# ------------------------------------------------------------------------------------------------
def sem_seg_postprocess(result, img_size, out_h, out_w):
    result = result[:, : img_size[0], : img_size[1]].expand(1, -1, -1, -1)
    return F.interpolate(result, size=(out_h, out_w), mode="bilinear", align_corners=False)[0]


def semantic_inference(cls, mask_pred):  # LP:402-406
    return torch.einsum("qc,qhw->chw", F.softmax(cls, dim=-1)[:, :-1], mask_pred.sigmoid())


def instance_inference(cls, mask_pred, topk, is_thing_list=None, panoptic_on=False):  # LP:407-447
    scores = F.softmax(cls, dim=-1)[:, :-1]
    nq, nc = scores.shape
    labels = torch.arange(nc).unsqueeze(0).repeat(nq, 1).flatten(0, 1)
    s, idx = scores.flatten(0, 1).topk(topk, sorted=False)
    lab = labels[idx]
    qi = idx // nc
    mp = mask_pred[qi]
    if panoptic_on:
        keep = torch.tensor([bool(is_thing_list[int(l)]) for l in lab])
        s, lab, mp, qi = s[keep], lab[keep], mp[keep], qi[keep]
    pm = (mp > 0).float()
    ms = (mp.sigmoid().flatten(1) * pm.flatten(1)).sum(1) / (pm.flatten(1).sum(1) + 1e-6)
    return dict(pred_masks=pm, scores=s * ms, pred_classes=lab, query_index=qi)


def seg_instance_inference(SEG_cls, mask_pred, topk):  # LP:308-324
    scores = torch.sigmoid(SEG_cls)
    s, idx = scores.flatten(0, 1).topk(topk, sorted=False)
    mp = mask_pred[idx]
    pm = (mp > 0).float()
    ms = (mp.sigmoid().flatten(1) * pm.flatten(1)).sum(1) / (pm.flatten(1).sum(1) + 1e-6)
    return dict(pred_masks=pm, scores=s * ms, query_index=idx)


def region_inference(region_cls, mask_pred):  # LP:387-400
    pm = (mask_pred > 0).float()
    mask_scores = (mask_pred.sigmoid().flatten(1) * pm.flatten(1)).sum(1) / (pm.flatten(1).sum(1) + 1e-6)
    scores = (region_cls.sigmoid() * mask_scores[None, ...].repeat(region_cls.shape[0], 1)).transpose(1, 0)
    return dict(pred_masks=pm, scores=scores)


def panoptic_inference(cls, mask_pred, is_thing_list, obj_thr=0.8, ovl_thr=0.8):  # LP:325-386
    scores, labels = F.softmax(cls, dim=-1).max(-1)
    nc = cls.shape[-1] - 1
    mp = mask_pred.sigmoid()
    keep = labels.ne(nc) & (scores > obj_thr)
    cs, cc, cm = scores[keep], labels[keep], mp[keep]
    h, w = cm.shape[-2:]
    pan = torch.zeros((h, w), dtype=torch.int32)
    info = []
    if cm.shape[0] == 0:
        return pan, info
    ids = (cs.view(-1, 1, 1) * cm).argmax(0)
    cur = 0
    stuff = {}
    for k in range(cc.shape[0]):
        pc = int(cc[k])
        isthing = is_thing_list[pc]
        area = int((ids == k).sum())
        orig = int((cm[k] >= 0.5).sum())
        m = (ids == k) & (cm[k] >= 0.5)
        if area > 0 and orig > 0 and int(m.sum()) > 0:
            if area / orig < ovl_thr:
                continue
            if not isthing:
                if pc in stuff:
                    pan[m] = stuff[pc]
                    continue
                stuff[pc] = cur + 1
            cur += 1
            pan[m] = cur
            info.append(dict(id=cur, isthing=bool(isthing), category_id=pc))
    return pan, info


# ------------------------------------------------------------------------------------------------
# eval_seg — LP:1317-1472
# ------------------------------------------------------------------------------------------------
def eval_seg(sd, input_ids, attention_mask, images, seg_info, class_name_ids=None, cls_indices=None,
             class_name_embedding_indices=None, token_refer_id=None, refer_embedding_indices=None,
             is_thing_list=None, task="panoptic", phi_cfg=PHI_15, return_intermediates=False,
             obj_thr=0.8, ovl_thr=0.8, region_points=None, vp_images=None):
    """Returns list (one dict per image).  NOTE the reference returns after image 0 (LP:1472);
    we process every image the same way.  obj_thr / ovl_thr: the panoptic thresholds the reference hard-codes
    to 0.8 / 0.8 (LP:331-332); other values only in accuracy runs on random weights (oracle/accuracy.py).
    vp_images: the DAVIS variant (PSALMForDAVISEval, LP:1477-1520, :1662-1670): the region features are pooled from the
    projector map of a SECOND image (the visual-prompt frame) with `instances.vp_region_masks`."""
    feats = swin_forward(sd, "model.vision_tower.", images)  # the reference runs this twice (LP:449, LP:223)
    img_tok = projector_forward(sd, "model.mm_projector.", feats[3])
    region_features = None
    if bool((input_ids == REGION_TOKEN_INDEX).any()):   # LP:1346-1349, LP:791-797
        # region_points: per sample [K,256,2]; None = draw them here from the global CPU generator like the reference
        attr = "region_masks" if vp_images is None else "vp_region_masks"   # LP:792 / LP:1664
        if region_points is None:
            region_points = [sample_region_points(getattr(info["instances"], attr).tensor) for info in seg_info]
        src_tok = img_tok
        if vp_images is not None:   # LP:1665
            src_tok = projector_forward(sd, "model.mm_projector.", swin_forward(sd, "model.vision_tower.", vp_images)[3])
        region_features = [region_pool(src_tok[b], region_points[b]) for b in range(images.shape[0])]
    seq = assemble_sequence(sd, input_ids, attention_mask, img_tok, class_name_ids, cls_indices,
                            class_name_embedding_indices, token_refer_id, refer_embedding_indices, region_features)
    hidden = phi_forward(sd, "model.", seq["inputs_embeds"], seq["attention_mask"], phi_cfg)
    seg_query = _lin(sd, "seg_query_projector", get_seg_query(hidden, seq["seg_query_mask"]))
    fd = dict(res2=feats[0], res3=feats[1], res4=feats[2], res5=feats[3])
    mask_features, _, ms = pixel_decoder_forward(sd, "pixel_decoder.", fd)
    SEG_emb = cls_emb = None
    if seq["refer_embedding_indices"] is not None:
        SEG_emb = _lin(sd, "SEG_token_projector", get_SEG_embedding(hidden, seq["refer_embedding_indices"]))
    if seq["class_name_embedding_indices"] is not None:
        cls_emb = _lin(sd, "class_name_projector", get_class_name_embedding(hidden, seq["class_name_embedding_indices"]))
    region_emb = None
    if seq["region_embedding_masks"] is not None:   # LP:1385-1388, LP:302-307
        region_emb = [_lin(sd, "region_projector", h[m.bool()]) for h, m in zip(hidden, seq["region_embedding_masks"])]
    po = predictor_forward(sd, "predictor.", ms, mask_features, seg_query, SEG_emb, cls_emb,
                           return_all=return_intermediates, region_embedding_list=region_emb)
    Hi, Wi = images.shape[-2:]
    Hp, Wp = (Hi + 31) // 32 * 32, (Wi + 31) // 32 * 32  # ImageList.from_tensors(size_divisibility=32) LP:1400
    mask_pred = F.interpolate(po["pred_masks"], size=(Hp, Wp), mode="bilinear", align_corners=False)
    results = []
    for b in range(images.shape[0]):
        info = seg_info[b]
        height, width = info.get("height", Hi), info.get("width", Wi)
        nz = np.where(~np.array(info["padding_mask"]))
        oh = int(nz[0].max() - nz[0].min() + 1)
        ow = int(nz[1].max() - nz[1].min() + 1)
        mp = mask_pred[b]
        r = {}
        before = task in ("instance", "panoptic", "referring", "region")  # LP:299
        if before:
            mp = sem_seg_postprocess(mp, (oh, ow), height, width)
        if task in ("semantic", "panoptic"):
            sem = semantic_inference(po["pred_class_name_logits"][b].float(), mp.float())
            if not before:
                sem = sem_seg_postprocess(sem, (oh, ow), height, width)
            r["sem_seg"] = sem
        if task in ("instance", "panoptic"):
            r["instances"] = instance_inference(po["pred_class_name_logits"][b].float(), mp.float(),
                                                po["pred_masks"].shape[1], is_thing_list, task == "panoptic")
        if task == "panoptic":
            r["panoptic_seg"] = panoptic_inference(po["pred_class_name_logits"][b].float(), mp.float(), is_thing_list,
                                                   obj_thr, ovl_thr)
        if task == "referring":
            r["instances"] = seg_instance_inference(po["pred_SEG_logits"][b].float(), mp.float(),
                                                    po["pred_masks"].shape[1])
        if task == "region":   # LP:1457-1466 (the reference indexes region_cls_results[0]: it returns after image 0)
            r["instances"] = region_inference(po["pred_region_logits"][b].float(), mp.float())
            r["gt"] = sem_seg_postprocess(info["instances"].gt_masks, (oh, ow), height, width)
        results.append(r)
    if return_intermediates:
        return results, dict(feats=feats, img_tok=img_tok, seq=seq, hidden=hidden, seg_query=seg_query,
                             mask_features=mask_features, ms=ms, SEG_emb=SEG_emb, cls_emb=cls_emb, predictor=po,
                             mask_pred=mask_pred, region_features=region_features, region_emb=region_emb,
                             region_points=region_points)
    return results
