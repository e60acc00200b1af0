"""Resampling kernels on the probes of tests/resample_probe.py: MSDeformAttn (vector kernel with the patch and the
linear query mapping, scalar kernel, device-side level shapes, fused encoder kernel), bilinear_tokens (scalar and
vector kernels), region_pool, and the task heads under psalm_set_postproc_impl 1 (generic) and 2 (tensor-core), plus
the composed crop path.

Exact probes compare with torch.equal against the float64 reference rounded once to storage; output buffers are
poisoned first (NaN / all-ones bits), so an unwritten element, row or slot shows.  Float64 probes stay within the
per-element bounds derived in tests/resample_probe.py.  Also: the MSDA dispatch on a contiguous `loc` / `w` with a
storage offset (the float4 preload needs 16-byte alignment), and the fused kernel's rejection of misaligned pointers.

Largest err / bound observed on an NVIDIA H100 80GB HBM3 (700 W power limit); every exact probe was bit-exact:
  fused MSDA, non-power-of-two levels      fp32 0.051   bf16 0.986 (the output rounding)
  bilinear_tokens, non-power-of-two        fp32 0.162   bf16 0.984
  task heads sum(sigma [x > 0])            generic 0.011   tensor-core 0.047
  task heads sem_seg                       0.718 (Q = 1), 0.111 otherwise
The whole file runs in about 20 s on that GPU."""
import contextlib
import ctypes
import math

import pytest
import torch

import resample_probe as rp
from psalm_b200 import _lib, kernels, msda

pytestmark = pytest.mark.gpu
CUDA = torch.device("cuda")
F64 = torch.float64
BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@contextlib.contextmanager
def _poisoned(*shapes_dtypes):
    """Fill the allocator's next blocks of these sizes with 0xFF bytes (NaN in every float type), so the kernel under
    test must overwrite every element it owns; yields the block addresses."""
    blocks = [torch.full((math.prod(s) * torch.empty((), dtype=d).element_size(),), 255, dtype=torch.uint8, device=CUDA)
              for s, d in shapes_dtypes]
    ptrs = {b.data_ptr() for b in blocks}
    del blocks
    yield ptrs


def _check_poisoned(t, ptrs):
    assert t.data_ptr() in ptrs, "the output did not reuse the poisoned block"


def _same(out, ref_stored):
    return torch.equal(out.to(F64), ref_stored.to(out.device))


# ---------------------------------------------------------------------------------------------------------------
# MSDeformAttn: vector / scalar kernels
# ---------------------------------------------------------------------------------------------------------------
MSDA_CASES = [  # shapes, M, D, value dtype, loc dtype, P, layout, linear Lq (0: Lq == S), device shapes
    ([(8, 16), (16, 16), (4, 8)], 8, 32, BF16, F32, 4, 0, 0, False),     # G 4, template (3, 4), preload, patch
    ([(8, 16), (16, 16), (4, 8), (2, 2)], 2, 16, BF16, F32, 4, 1, 0, False),   # G 2, (4, 4), head-major
    ([(8, 8), (16, 16), (32, 32)], 4, 4, F32, F32, 4, 0, 0, False),    # G 1
    ([(16, 16), (8, 8)], 1, 128, F32, F32, 3, 0, 0, False),             # G 32, runtime (2, 3)
    ([(16, 16), (8, 8)], 2, 256, BF16, BF16, 3, 1, 0, False),           # G 32, bf16 loc
    ([(8, 16), (16, 16), (4, 8)], 3, 128, F16, F16, 4, 0, 77, False),   # G 16, 16-bit loc, linear mapping
    ([(16, 8)], 2, 64, BF16, F32, 1, 0, 50, False),                     # G 8, (1, 1)... P = 1
    ([(5, 7), (11, 13)], 2, 32, F32, F32, 2, 0, 0, False),              # odd levels, G 8
    ([(5, 7), (11, 13), (3, 4)], 2, 8, BF16, F32, 4, 1, 0, True),        # device shapes, G 1
    ([(8, 16), (16, 16), (4, 8)], 2, 32, F32, F32, 4, 0, 0, True),       # device shapes, template
    ([(8, 16), (16, 16)], 2, 2, F32, F32, 4, 0, 0, False),              # scalar: D = 2
    ([(5, 7), (11, 13)], 3, 6, BF16, BF16, 3, 1, 40, False),            # scalar: D = 6, linear
    ([(8, 16), (16, 16), (4, 8)], 1, 256, F32, F32, 4, 0, 0, False),     # scalar: fp32 D = 256 (G = 64)
]


def _msda_inputs(value, shapes, layout, device_shapes):
    """(value in `layout`, level shapes, level starts) as the op takes them; built before any poisoning."""
    v = value if layout == 0 else value.permute(0, 2, 1, 3).contiguous()
    starts = rp.level_starts(shapes)
    if device_shapes:
        return (v, torch.tensor(shapes, dtype=torch.int64, device=CUDA),
                torch.tensor(starts, dtype=torch.int64, device=CUDA))
    return v, shapes, starts


def _run_msda(value, shapes, loc, aw, layout, device_shapes):
    v, sh, st = _msda_inputs(value, shapes, layout, device_shapes)
    return msda.ms_deform_attn_forward(v, sh, st, loc, aw, 128, layout)


@pytest.mark.parametrize("case", range(len(MSDA_CASES)))
def test_msda_exact_probe(case):
    shapes, M, D, vdt, ldt, P, layout, Lq, dev_shapes = MSDA_CASES[case]
    B = 2
    S = sum(h * w for h, w in shapes)
    Lq = Lq or S
    value = rp.msda_value(B, shapes, M, D, CUDA)
    loc, aw = rp.msda_probe(B, shapes, M, Lq, P, _gen(case), ldt, CUDA)
    ref = rp.stored(rp.msda_ref(value, shapes, loc, aw), vdt)
    v, sh, st = _msda_inputs(value.to(vdt), shapes, layout, dev_shapes)
    loc, aw = loc.to(ldt), aw.to(ldt)
    with _poisoned(((B, Lq, M * D), vdt)) as ptrs:
        out = msda.ms_deform_attn_forward(v, sh, st, loc, aw, 128, layout)
    _check_poisoned(out, ptrs)
    assert _same(out, ref)


@pytest.mark.parametrize("dtype", [BF16, F32])
def test_msda_full_size_exact(dtype):
    """The pixel decoder at 1024^2: S = 21504 queries, M = 8, D = 32, levels 128 / 64 / 32, vector kernel (patch)."""
    shapes = [(128, 128), (64, 64), (32, 32)]
    M, D = 8, 32
    S = sum(h * w for h, w in shapes)
    value = rp.msda_value(1, shapes, M, D, CUDA)
    loc, aw = rp.msda_probe(1, shapes, M, S, 4, _gen(11), F32, CUDA)
    ref = rp.stored(rp.msda_ref(value, shapes, loc, aw), dtype)
    out = _run_msda(value.to(dtype), shapes, loc.float(), aw.float(), 0, False)
    assert _same(out, ref)


@pytest.mark.parametrize("LP", [(3, 4), (4, 4)])
def test_msda_loc_and_weights_with_a_storage_offset(LP):
    """Contiguous fp32 loc 8 bytes past a 16-byte boundary and w 4 bytes past one: the (3,4) / (4,4) instantiations
    must not preload them with float4 loads; the result is the reference's."""
    L, P = LP
    shapes = [(8, 16), (16, 16), (4, 8), (2, 4)][:L]
    B, M, D = 2, 8, 32
    S = sum(h * w for h, w in shapes)
    value = rp.msda_value(B, shapes, M, D, CUDA)
    loc, aw = rp.msda_probe(B, shapes, M, S, P, _gen(7), F32, CUDA)
    ref = rp.stored(rp.msda_ref(value, shapes, loc, aw), BF16)
    lbuf = torch.empty(loc.numel() + 2, dtype=F32, device=CUDA)[2:].view(loc.shape)
    wbuf = torch.empty(aw.numel() + 1, dtype=F32, device=CUDA)[1:].view(aw.shape)
    lbuf.copy_(loc)
    wbuf.copy_(aw)
    assert lbuf.is_contiguous() and lbuf.data_ptr() % 16 == 8 and wbuf.data_ptr() % 16 == 4
    out = _run_msda(value.to(BF16), shapes, lbuf, wbuf, 0, False)
    assert _same(out, ref)
    for dev_shapes, layout in ((True, 0), (False, 1)):
        assert _same(_run_msda(value.to(BF16), shapes, lbuf, wbuf, layout, dev_shapes), ref)


# ---------------------------------------------------------------------------------------------------------------
# MSDeformAttn: fused encoder kernel
# ---------------------------------------------------------------------------------------------------------------
FUSED_CASES = [  # shapes, hot, value dtype, ow dtype, D
    ([(16, 16), (8, 8), (4, 4)], 1, BF16, BF16, 32),          # G 4 (TH 8), ragged 4x4
    ([(16, 16), (8, 8), (4, 4)], 4, BF16, F32, 64),           # G 8 (TH 4)
    ([(8, 16), (4, 8), (2, 4), (1, 2)], 16, F32, F32, 16),   # G 4, L 4, 16-hot
    ([(8, 16), (4, 8), (2, 4), (1, 2)], 2, F32, F32, 32),    # G 8
    ([(16, 8), (8, 4), (4, 2)], 2, F16, F16, 32),
    ([(32, 16), (16, 8), (8, 4)], 1, F16, F32, 64),
]


def _run_fused(value_hm, ow, shapes):
    return msda.msda_encoder_fused(value_hm, ow, shapes, rp.level_starts(shapes))


@pytest.mark.parametrize("case", range(len(FUSED_CASES)))
def test_fused_exact_probe(case):
    shapes, hot, vdt, odt, D = FUSED_CASES[case]
    B, M = 2, 8
    S = sum(h * w for h, w in shapes)
    value = rp.msda_value(B, shapes, M, D, CUDA).permute(0, 2, 1, 3).contiguous()
    ow = rp.fused_probe(B, shapes, M, _gen(20 + case), hot, odt, device=CUDA)
    ref = rp.stored(rp.msda_fused_ref(value, ow, shapes), vdt)
    value, ow = value.to(vdt), ow.to(odt)
    with _poisoned(((B, S, M * D), vdt)) as ptrs:
        out = _run_fused(value, ow, shapes)
    _check_poisoned(out, ptrs)
    assert _same(out, ref)


@pytest.mark.parametrize("dtype", [BF16, F32])
def test_fused_full_size_exact(dtype):
    shapes = [(128, 128), (64, 64), (32, 32)]
    M, D = 8, 32
    value = rp.msda_value(1, shapes, M, D, CUDA).permute(0, 2, 1, 3).contiguous()
    ow = rp.fused_probe(1, shapes, M, _gen(30), 1, dtype, device=CUDA)
    ref = rp.stored(rp.msda_fused_ref(value, ow, shapes), dtype)
    assert _same(_run_fused(value.to(dtype), ow.to(dtype), shapes), ref)


WORST = {}


@pytest.mark.parametrize("dtype,D", [(F32, 16), (BF16, 64)])
def test_fused_float64_probe(dtype, D):
    shapes = [(13, 21), (7, 11), (4, 5)]
    B, M = 2, 8
    value = rp.msda_value(B, shapes, M, D, CUDA).permute(0, 2, 1, 3).contiguous()
    ow = rp.fused_probe(B, shapes, M, _gen(40), 2, F32, device=CUDA)
    ref = rp.msda_fused_ref(value, ow, shapes)
    bound = rp.fused_bound(value, ow, shapes, ref, dtype)
    out = _run_fused(value.to(dtype), ow.float(), shapes)
    r = rp.err_over_bound(out, ref, bound)
    print("fused float64 %s err/bound %.3f" % (dtype, r))
    assert r <= 1.0


def test_fused_rejects_misaligned_pointers():
    shapes = [(8, 8), (4, 4), (2, 2)]
    B, M, D = 1, 8, 32
    S = sum(h * w for h, w in shapes)
    value = rp.msda_value(B, shapes, M, D, CUDA).permute(0, 2, 1, 3).contiguous().to(BF16)
    ow = rp.fused_probe(B, shapes, M, _gen(50), 1, F32, device=CUDA).float()
    vbad = torch.empty(value.numel() + 2, dtype=BF16, device=CUDA)[2:].view(value.shape)     # 4 bytes off
    obad = torch.empty(ow.numel() + 1, dtype=F32, device=CUDA)[1:].view(ow.shape)            # 4 bytes off
    vbad.copy_(value)
    obad.copy_(ow)
    for v, o in ((vbad, ow), (value, obad)):
        with pytest.raises(RuntimeError, match="aligned"):
            _run_fused(v, o, shapes)
    out = torch.zeros(B * S * M * D + 8, dtype=BF16, device=CUDA)
    flat = [v for hw in shapes for v in hw]
    rc = _lib.lib().psalm_msda_encoder_fused(
        _lib.ptr(value), _lib.ptr(ow), ctypes.c_void_p(out.data_ptr() + 4), _lib.i64_array(flat),
        _lib.i64_array(rp.level_starts(shapes)), B, S, M, D, 3, 4, _lib.BF16, _lib.F32, _lib.stream_ptr(CUDA))
    assert rc != 0 and b"aligned" in _lib.lib().psalm_last_error()
    torch.cuda.synchronize()
    assert (out == 0).all()                                            # nothing launched
    assert _same(_run_fused(value, ow, shapes), rp.stored(rp.msda_fused_ref(value.double(), ow.double(), shapes), BF16))


# ---------------------------------------------------------------------------------------------------------------
# bilinear_tokens, region_pool
# ---------------------------------------------------------------------------------------------------------------
BIL_CASES = [(8, 12, 16, 24), (5, 7, 10, 14), (16, 12, 8, 6), (20, 28, 5, 7), (24, 16, 3, 2), (64, 64, 128, 128),
             (128, 128, 32, 32), (256, 256, 32, 32)]


@pytest.mark.parametrize("Hi,Wi,Ho,Wo", BIL_CASES)
@pytest.mark.parametrize("path", ["vec", "scalar_c", "scalar_f32out"])
@pytest.mark.parametrize("dtype", [BF16, F32])
def test_bilinear_exact_probe(Hi, Wi, Ho, Wo, path, dtype):
    if path == "scalar_f32out" and dtype == F32:
        pytest.skip("fp32 input has no wider output")
    B = 2
    C = {"vec": 16, "scalar_c": 6, "scalar_f32out": 16}[path]
    odt = F32 if path == "scalar_f32out" else dtype
    x = rp.tokens_probe(B, Hi, Wi, C, CUDA)
    xs = x.to(dtype)
    with _poisoned(((B, Ho * Wo, C), odt)) as ptrs:
        out = kernels.bilinear_tokens(xs, Hi, Wi, Ho, Wo, out_dtype=odt)
    _check_poisoned(out, ptrs)
    assert _same(out, rp.stored(rp.bilinear_ref(x, Hi, Wi, Ho, Wo), odt))
    old = rp.stored(rp.tokens_probe(B, Ho, Wo, C, CUDA).flip(-1) * 3, odt)
    acc = old.to(odt)
    kernels.bilinear_tokens(xs, Hi, Wi, Ho, Wo, out=acc, accumulate=True)
    assert _same(acc, rp.stored(rp.bilinear_ref(x, Hi, Wi, Ho, Wo, old), odt))


@pytest.mark.parametrize("Hi,Wi,Ho,Wo", [(24, 20, 37, 29), (15, 17, 40, 33), (64, 64, 100, 90), (37, 29, 24, 20)])
@pytest.mark.parametrize("C,dtype,odt", [(16, BF16, BF16), (6, BF16, F32), (16, F32, F32)])
def test_bilinear_float64_probe(Hi, Wi, Ho, Wo, C, dtype, odt):
    x = rp.tokens_probe(1, Hi, Wi, C, CUDA)
    ref = rp.bilinear_ref(x, Hi, Wi, Ho, Wo)
    out = kernels.bilinear_tokens(x.to(dtype), Hi, Wi, Ho, Wo, out_dtype=odt)
    r = rp.err_over_bound(out, ref, rp.bilinear_bound(x, Hi, Wi, ref, odt))
    print("bilinear float64 %s %s err/bound %.3f" % ((Hi, Wi, Ho, Wo), odt, r))
    assert r <= 1.0


@pytest.mark.parametrize("h,w", [(9, 17), (17, 33), (33, 9)])
@pytest.mark.parametrize("dtype,C", [(BF16, 16), (F32, 8), (F16, 32)])
def test_region_pool_exact_probe(h, w, dtype, C):
    tokens, pts, img = rp.region_probe(3, h, w, C, 7, 256, _gen(60), CUDA)
    ref = rp.stored(rp.region_ref(tokens, h, w, pts, img), dtype)
    tokens, pts = tokens.to(dtype), pts.float()
    with _poisoned(((7, C), dtype)) as ptrs:
        out = kernels.region_pool(tokens, pts, img, h, w)
    _check_poisoned(out, ptrs)
    assert _same(out, ref)


# ---------------------------------------------------------------------------------------------------------------
# task heads
# ---------------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _postproc_impl(v):
    fn = _lib.lib().psalm_set_postproc_impl
    _lib.check(fn(v), "psalm_set_postproc_impl")
    try:
        yield
    finally:
        fn(0)


def _heads_call(logits, H, W, probsT, wq, negq, slots, ncls, crop=None):
    """The C ABI with poisoned outputs: NaN sem / inst, -1 ids, 255 in_mask, NaN partials."""
    Q, H4, W4 = logits.shape
    K = slots.shape[0]
    rows = ctypes.c_int()
    if crop is None:
        _lib.check(_lib.lib().psalm_postproc_partials(Q, H4, W4, H, W, ncls, K, _lib.dtype_code(logits.dtype),
                                                      ctypes.byref(rows)), "psalm_postproc_partials")
    else:
        _lib.check(_lib.lib().psalm_postproc_crop_partials(H, W, ctypes.byref(rows)), "psalm_postproc_crop_partials")
    nan = float("nan")
    part = torch.full((rows.value, Q, 5), nan, device=CUDA)
    sem = torch.full((ncls, H, W), nan, device=CUDA) if probsT is not None else None
    ids = torch.full((H, W), -1, dtype=torch.int32, device=CUDA)
    inm = torch.full((H, W), 255, dtype=torch.uint8, device=CUDA)
    inst = torch.full((K, H, W), nan, device=CUDA)
    p = lambda t: _lib.ptr(t) if t is not None else None   # noqa: E731
    probs16 = probsT.to(CUDA, F16).contiguous() if probsT is not None else None
    sl = slots.to(CUDA, torch.int32).contiguous()
    wq, negq = wq.to(CUDA, F32).contiguous(), negq.to(CUDA, F32).contiguous()
    assert logits.is_cuda
    args = (p(logits), p(probs16), p(wq), p(negq), p(sl), p(sem), p(inst), p(ids), p(inm), p(part))
    if crop is None:
        rc = _lib.lib().psalm_postproc_fused(*args, Q, H4, W4, H, W, ncls, K, _lib.dtype_code(logits.dtype),
                                             _lib.stream_ptr(CUDA))
    else:
        Hp, Wp, oh, ow = crop
        rc = _lib.lib().psalm_postproc_fused_crop(*args, Q, H4, W4, Hp, Wp, oh, ow, H, W, ncls, K,
                                                  _lib.dtype_code(logits.dtype), _lib.stream_ptr(CUDA))
    _lib.check(rc, "psalm_postproc_fused")
    return dict(stats=part.sum(0).double(), sem=sem, ids=ids, in_mask=inm, inst=inst, rows=rows.value)


def _check_heads(got, ref, slots, fast):
    """Exact outputs equal; a pixel whose panoptic winner leads by less than IDS_MARGIN may take any query within the
    margin, and in_mask / area / intersection then follow the kernel's choice exactly."""
    st, rs = got["stats"], ref["stats"]
    for col in (0, 2):
        assert torch.equal(st[:, col], rs[:, col]), col
    ids = got["ids"].long()
    clear = ref["ids_clear"]
    assert torch.equal(ids[clear], ref["ids"][clear])
    assert bool(ref["ids_cand"].gather(0, ids.unsqueeze(0)).all())
    inm = (ref["x"].gather(0, ids.unsqueeze(0))[0] >= 0).to(torch.uint8)
    assert torch.equal(got["in_mask"], inm)
    Q = st.shape[0]
    assert torch.equal(st[:, 3], torch.bincount(ids.flatten(), minlength=Q).double())
    assert torch.equal(st[:, 4], torch.bincount(ids.flatten(), weights=inm.flatten().double(), minlength=Q))
    if bool(clear.all()):
        assert torch.equal(st[:, 3:], rs[:, 3:]) and torch.equal(got["in_mask"], ref["in_mask"])
    has = (slots >= 0).to(CUDA)
    assert torch.equal(got["inst"][has].double(), ref["inst"][has])
    bound = ref["sig_bound_fast"] if fast else ref["sig_bound_generic"]
    r_sig = ((st[:, 1] - rs[:, 1]).abs() / bound.clamp_min(1e-30)).max().item()
    r_sem = rp.err_over_bound(got["sem"], ref["sem"], ref["sem_bound"]) if got["sem"] is not None else 0.0
    return r_sig, r_sem


HEADS_CASES = [  # Q, H4, W4, ratio, ncls, K, logits dtype
    (37, 12, 10, 4, 47, 100, BF16),
    (104, 8, 6, 8, 133, 256, F16),
    (100, 20, 18, 4, 48, 256, BF16),
    (112, 3, 22, 8, 144, 1, BF16),      # Q 112: tensor-core kernel only
    (1, 12, 10, 4, 1, 1, BF16),
    (100, 21, 17, 4, 134, 257, BF16),   # odd W4, K 257: generic only
    (104, 8, 6, 8, 133, 100, F32),      # fp32 logits: generic only
]


@pytest.mark.parametrize("case", range(len(HEADS_CASES)))
@pytest.mark.parametrize("impl", [1, 2])
def test_heads_exact_probe(case, impl):
    Q, H4, W4, ratio, ncls, K, dt = HEADS_CASES[case]
    H, W = H4 * ratio, W4 * ratio
    # x1 / x2 up-sampling needs more source taps per 8 x 16 tile than either kernel stages: both refuse it
    fast_ok = dt != F32 and Q <= 112 and K <= 256 and W4 % 2 == 0 and ratio >= 4
    generic_ok = Q <= 104 and ratio >= 4
    if (impl == 2 and not fast_ok) or (impl == 1 and not generic_ok):
        pytest.skip("path does not take this geometry")
    logits, probsT, wq, negq, slots = rp.heads_probe(Q, H4, W4, ratio, ncls, K, device=CUDA)
    x = rp.heads_x(logits, H, W)
    with _postproc_impl(impl):
        got = _heads_call(logits.to(dt), H, W, probsT, wq, negq, slots, ncls)
    ref = rp.heads_ref(x, probsT, wq, negq, slots, ncls, rows=got["rows"])
    props = rp.probe_properties(x, ref, Q)
    assert props["decided"] and props["zero_rows"] and props["zero_free_rows"] and (props["tie_wins"] or Q <= 11)
    r_sig, r_sem = _check_heads(got, ref, slots, impl == 2)
    print("heads impl %d case %d: sum(sigma) err/bound %.3f, sem %.3f, %d pixels within the ids margin"
          % (impl, case, r_sig, r_sem, int((~ref["ids_clear"]).sum())))
    assert r_sig <= 1.0 and r_sem <= 1.0


@pytest.mark.parametrize("dt", [BF16, F32])
def test_heads_composed_exact_probe(dt):
    Q, H4, W4, ncls, K = 37, 10, 12, 47, 100
    crop, H, W = (40, 48, 36, 40), 72, 80
    assert kernels.postproc_crop_supported(Q, H4, W4, *crop, H, W, ncls)
    logits, probsT, wq, negq, slots = rp.heads_probe(Q, H4, W4, 4, ncls, K, device=CUDA)
    x = rp.heads_x(logits, H, W, crop)
    got = _heads_call(logits.to(dt), H, W, probsT, wq, negq, slots, ncls, crop)
    ref = rp.heads_ref(x, probsT, wq, negq, slots, ncls, rows=got["rows"])
    assert bool(ref["ids_clear"].all())
    r_sig, r_sem = _check_heads(got, ref, slots, False)
    assert r_sig <= 1.0 and r_sem <= 1.0


CROP_GEOMETRIES = {  # H4, W4, Hp, Wp, oh, ow, H, W: tests/test_postprocess.py's composed crop geometries
    "down": (64, 64, 256, 256, 192, 256, 120, 160),
    "up": (48, 64, 192, 256, 150, 200, 300, 400),
    "portrait": (64, 64, 256, 256, 256, 171, 640, 427),
    "coco-1024": (256, 256, 1024, 1024, 768, 1024, 480, 640),
}


@pytest.mark.parametrize("geom", list(CROP_GEOMETRIES))
@pytest.mark.parametrize("dt", [BF16, F32])
def test_heads_composed_float64_probe(geom, dt):
    """The composed crop path at non-power-of-two resize ratios: exact outside the flip sets the bound allows, sem_seg
    and sum(sigma [x > 0]) within their bounds (tests/resample_probe.py, crop_violations)."""
    H4, W4, Hp, Wp, oh, ow, H, W = CROP_GEOMETRIES[geom]
    Q, ncls, K = 100, 133, 100
    crop = (Hp, Wp, oh, ow)
    assert kernels.postproc_crop_supported(Q, H4, W4, *crop, H, W, ncls)
    logits, probsT, wq, negq, slots = rp.heads_probe(Q, H4, W4, 4, ncls, K, device=CUDA)
    bx = rp.crop_x_bound(logits, crop, H, W)
    got = _heads_call(logits.to(dt), H, W, probsT, wq, negq, slots, ncls, crop)
    ref = rp.heads_ref(rp.heads_x(logits, H, W, crop), probsT, wq, negq, slots, ncls, rows=got["rows"])
    assert rp.crop_violations(got, ref, probsT, ncls, slots, bx) == []
    x = ref["x"]
    P = probsT[:ncls, :Q]
    sem_b = ref["sem_bound"] + (P * (bx / 4)).sum(1).view(-1, 1, 1)
    r_sem = rp.err_over_bound(got["sem"], ref["sem"], sem_b)
    npos, nflip = (x > -bx).flatten(1).sum(1), (x.abs() <= bx).flatten(1).sum(1)
    sig_b = ref["sig_bound_generic"] + npos * bx / 4 + nflip * (0.5 + bx / 4)
    r_sig = ((got["stats"][:, 1] - ref["stats"][:, 1]).abs() / sig_b).max().item()
    print("heads crop %s %s: bx %.2e, %d pixels may flip, sum(sigma) err/bound %.3f, sem %.3f"
          % (geom, dt, bx, int(nflip.sum()), r_sig, r_sem))


@pytest.mark.parametrize("impl", [0, 1])
def test_heads_full_size(impl):
    """256^2 logits -> 1024^2, Q = 100, ncls = 134, K = 100, bf16: the benchmark's geometry (impl 0 takes the
    tensor-core kernel there)."""
    Q, H4, ncls, K = 100, 256, 134, 100
    logits, probsT, wq, negq, slots = rp.heads_probe(Q, H4, H4, 4, ncls, K, device=CUDA)
    with _postproc_impl(impl):
        got = _heads_call(logits.to(BF16), 1024, 1024, probsT, wq, negq, slots, ncls)
    x = rp.heads_x(logits, 1024, 1024)
    ref = rp.heads_ref(x, probsT, wq, negq, slots, ncls, rows=got["rows"])
    del x
    assert (~ref["ids_clear"]).float().mean() < 1e-5
    r_sig, r_sem = _check_heads(got, ref, slots, impl != 1)
    print("heads full size impl %d: sum(sigma) err/bound %.3f, sem %.3f, %d pixels within the ids margin"
          % (impl, r_sig, r_sem, int((~ref["ids_clear"]).sum())))
    assert r_sig <= 1.0 and r_sem <= 1.0


def test_heads_fast_kernel_at_its_largest_tile_count():
    """Constant-logit maps at the largest tile count per CTA the tensor-core kernel admits (255, from the device's SM
    count): every count is H W or 0, a saturated map's sum(sigma) is exactly H W (sigma = 1 in fp32), the others
    H W sigma(c) within the bound; one more tile row per CTA is refused by the forced tensor-core path, and the
    automatic routing gives the same results on the generic kernel."""
    consts = [127, 127, -127, 0, 5, -3, 127, 2]
    Q = len(consts)
    kept = torch.tensor([1, 1, 1, 1, 1, 1, 0, 1], dtype=torch.bool)
    wq = torch.tensor([0.75, 0.75, 0.5, 0.5, 0.5, 0.5, 0.0, 0.25], dtype=F64)
    negq = torch.where(kept, torch.zeros(Q, dtype=F64), -torch.ones(Q, dtype=F64))
    slots = torch.tensor([0, 3, -1, 4, 2, 0], dtype=torch.int64)
    probsT = torch.zeros(144, 112, dtype=F64)
    probsT[0, :Q] = torch.arange(1, Q + 1, dtype=F64) / 64
    probsT[1, :Q] = 0.125
    sig = torch.tensor([rp.sigmoid(c) for c in consts], dtype=F64)
    H4, W4, H, W = rp.fast_max_tiles_geometry(_sms())
    for impl, extra_row in ((2, False), (0, True)):
        Hx, Hx4 = (H + 64, H4 + 8) if extra_row else (H, H4)      # 8 more tile rows: 263 tiles per CTA
        logits = rp.constant_heads(Q, Hx4, W4, consts, CUDA).to(BF16)
        with _postproc_impl(impl):
            got = _heads_call(logits, Hx, W, probsT, wq, negq, slots, 2)
        n = Hx * W
        st = got["stats"].cpu()
        c = torch.tensor(consts, dtype=F64)
        assert torch.equal(st[:, 0], (c > 0).to(F64) * n)
        assert torch.equal(st[:, 2], (c >= 0).to(F64) * n)
        assert torch.equal(st[:, 3], torch.tensor([n] + [0] * (Q - 1), dtype=F64))
        assert torch.equal(st[:, 4], st[:, 3])
        sat = c == 127
        assert torch.equal(st[sat, 1], torch.full((int(sat.sum()),), float(n), dtype=F64))
        want = sig * n * (c > 0)
        bound = n * 2.0 ** -11 * 1.01 + (129 + got["rows"]) * rp.U32 * want
        assert ((st[:, 1] - want).abs() <= bound).all()
        assert bool((got["ids"] == 0).all()) and bool((got["in_mask"] == 1).all())
        for k, q in enumerate(slots.tolist()):
            if q >= 0:
                assert bool((got["inst"][k] == float(consts[q] > 0)).all()), k
        got["ids"] = got["inst"] = None
        sem_want = (probsT[:2, :Q] * sig).sum(1)
        for cl in range(2):
            e = (got["sem"][cl].double() - sem_want[cl]).abs().max().item()
            assert e <= (2.0 ** -11 + 2.0 ** -15) * sem_want[cl] + 2.0 ** -19 * probsT[cl].sum() + rp.U32 * sem_want[cl]
        del got
    with _postproc_impl(2):
        with pytest.raises(_lib.PsalmKernelError, match="tensor-core path forced but unsupported"):
            _heads_call(rp.constant_heads(Q, H4 + 8, W4, consts, CUDA).to(BF16), H + 64, W, probsT, wq, negq, slots, 2)
