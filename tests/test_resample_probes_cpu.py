"""The resampling probes of tests/resample_probe.py can fail: each exact probe's reference is exact in storage and
differs from every named mutant in at least one bit, and each float64 probe misses every named mutant by >= 10x the
bound that tests/test_resample_probes_gpu.py applies to the kernels.  The fast task-head kernel's wrapping fixed-point
accumulation is emulated at its largest tile count.  No kernel runs here."""
import pytest
import torch

import resample_probe as rp

F64 = torch.float64
DT16 = [torch.bfloat16, torch.float16]


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _differs(a, b):
    return not torch.equal(a, b)


def _exact(ref, dtype):
    return torch.equal(rp.stored(ref, dtype), ref)


def _missed(mut, ref, bound):
    d = (mut - ref).abs() / bound
    d = torch.where(torch.isnan(d), torch.full_like(d, float("inf")), d)
    return d.max().item() >= 10


# ---------------------------------------------------------------------------------------------------------------
# MSDeformAttn
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shapes,P,loc_dtype", [
    ([(8, 16), (16, 16), (4, 8)], 4, torch.float32),
    ([(16, 16), (8, 8), (4, 4), (2, 2)], 4, torch.float32),
    ([(8, 8), (16, 8)], 3, torch.bfloat16),
    ([(5, 7), (11, 13)], 2, torch.float32),
    ([(5, 7), (11, 13), (3, 4)], 4, torch.float16),
])
def test_msda_probe_is_exact_and_rejects_mutants(shapes, P, loc_dtype):
    B, M, D = 2, 3, 4
    S = sum(h * w for h, w in shapes)
    value = rp.msda_value(B, shapes, M, D)
    loc, aw = rp.msda_probe(B, shapes, M, S, P, _gen(1), loc_dtype)
    assert torch.equal(rp.stored(loc, loc_dtype), loc) and value.abs().max() <= 125
    ref = rp.msda_ref(value, shapes, loc, aw)
    for dt in DT16 + [torch.float32]:
        st = lambda t: rp.stored(t, dt)          # noqa: E731
        if dt == torch.float32:
            assert _exact(ref, dt)
        for mut in rp.MSDA_MUTANTS:
            assert _differs(st(rp.msda_ref(value, shapes, loc, aw, mut)), st(ref)), (mut, dt)


def test_msda_equivalent_mutants_equal_the_reference():
    """At x = -1 (x = W) the one corner inside the map has bilinear weight 0, so `>= -1` / `<= W` compute the same
    result as `> -1` / `< W` on a probe that samples exactly there, in both axes."""
    shapes = [(8, 16), (16, 16)]
    value = rp.msda_value(2, shapes, 2, 4)
    loc, aw = rp.msda_probe(2, shapes, 2, 200, 4, _gen(2))
    for l, (h, w) in enumerate(shapes):
        assert bool(((loc[..., l, :, 0] * w - 0.5) == -1).any()) and bool(((loc[..., l, :, 0] * w - 0.5) == w).any())
        assert bool(((loc[..., l, :, 1] * h - 0.5) == -1).any()) and bool(((loc[..., l, :, 1] * h - 0.5) == h).any())
    ref = rp.msda_ref(value, shapes, loc, aw)
    for mut in rp.MSDA_EQUIVALENT:
        assert torch.equal(rp.msda_ref(value, shapes, loc, aw, mut), ref), mut


def test_msda_probe_hits_every_edge_case():
    shapes = [(8, 16), (16, 16)]
    loc, _ = rp.msda_probe(1, shapes, 2, 200, 4, _gen(2))
    for l, (h, w) in enumerate(shapes):
        xs = set((loc[..., l, :, 0] * w - 0.5).flatten().tolist())
        ys = set((loc[..., l, :, 1] * h - 0.5).flatten().tolist())
        assert set(rp.edge_positions(w)) <= xs and set(rp.edge_positions(h)) <= ys


@pytest.mark.parametrize("shapes,hot,ow_dtype", [
    ([(16, 16), (8, 8), (4, 4)], 1, torch.float32),
    ([(8, 16), (4, 8), (2, 4), (1, 2)], 16, torch.float32),
    ([(16, 8), (8, 4), (4, 2)], 2, torch.bfloat16),
    ([(4, 4), (2, 2), (2, 1)], 4, torch.float16),
])
def test_fused_probe_is_exact_and_rejects_mutants(shapes, hot, ow_dtype):
    B, M, D = 2, 8, 4
    value = rp.msda_value(B, shapes, M, D).permute(0, 2, 1, 3).contiguous()
    ow = rp.fused_probe(B, shapes, M, _gen(3), hot, ow_dtype)
    ref = rp.msda_fused_ref(value, ow, shapes)
    # exact in storage up to the e^-200 weights of the "cold" logits
    assert (ref - rp.stored(ref, torch.float32)).abs().max() < 1e-60
    st = lambda t: rp.stored(t, torch.bfloat16)                 # noqa: E731
    for mut in rp.FUSED_MUTANTS:
        if mut == "ragged_wrap" and all(w % rp.MSDA_TW == 0 for _, w in shapes):
            continue
        if mut == "softmax_per_level" and hot == 1:
            continue   # a one-hot head has one live level: a per-level softmax differs only in the cold levels
        assert _differs(st(rp.msda_fused_ref(value, ow, shapes, mutant=mut)), st(ref)), mut


def test_fused_float64_probe_misses_mutants_by_10x():
    shapes = [(13, 21), (7, 11), (4, 5)]
    value = rp.msda_value(1, shapes, 8, 4).permute(0, 2, 1, 3).contiguous()
    ow = rp.fused_probe(1, shapes, 8, _gen(4), 2)
    ref = rp.msda_fused_ref(value, ow, shapes)
    for dt in (torch.float32, torch.bfloat16):            # every bound the GPU file applies
        bound = rp.fused_bound(value, ow, shapes, ref, dt)
        for mut in rp.FUSED_MUTANTS:
            assert _missed(rp.msda_fused_ref(value, ow, shapes, mutant=mut), ref, bound), (mut, dt)


# ---------------------------------------------------------------------------------------------------------------
# bilinear_tokens, region_pool
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Hi,Wi,Ho,Wo", [(8, 12, 16, 24), (5, 7, 10, 14), (16, 12, 8, 6), (20, 28, 5, 7),
                                         (24, 16, 3, 2), (32, 40, 4, 5)])
def test_bilinear_probe_is_exact_and_rejects_mutants(Hi, Wi, Ho, Wo):
    x = rp.tokens_probe(2, Hi, Wi, 6)
    old = rp.tokens_probe(2, Ho, Wo, 6).flip(-1) * 3
    for acc in (None, old):
        ref = rp.bilinear_ref(x, Hi, Wi, Ho, Wo, acc)
        assert _exact(ref, torch.float32)
        for dt in DT16:
            st = lambda t: rp.stored(t, dt)        # noqa: E731
            for mut in rp.BILINEAR_MUTANTS:
                if mut == "accumulate_drops_old" and acc is None:
                    continue
                if Ho < Hi and Wo < Wi and mut in ("no_clamp", "upper_unclamped"):
                    # down-sampling never has a negative source index nor an upper tap past the map: equivalent
                    assert torch.equal(rp.bilinear_ref(x, Hi, Wi, Ho, Wo, acc, mut), ref)
                    continue
                assert _differs(st(rp.bilinear_ref(x, Hi, Wi, Ho, Wo, acc, mut)), st(ref)), (mut, dt)


@pytest.mark.parametrize("Hi,Wi,Ho,Wo", [(24, 20, 37, 29), (15, 17, 40, 33), (64, 64, 100, 90), (37, 29, 24, 20)])
def test_bilinear_float64_probe_misses_mutants_by_10x(Hi, Wi, Ho, Wo):
    x = rp.tokens_probe(1, Hi, Wi, 6)
    ref = rp.bilinear_ref(x, Hi, Wi, Ho, Wo)
    for dt in (torch.float32, torch.bfloat16):            # every bound the GPU file applies
        bound = rp.bilinear_bound(x, Hi, Wi, ref, dt)
        for mut in ("align_corners", "no_clamp", "upper_unclamped"):
            if Ho < Hi and Wo < Wi and mut in ("no_clamp", "upper_unclamped"):
                continue   # equivalent when down-sampling (test_bilinear_probe_is_exact_and_rejects_mutants)
            assert _missed(rp.bilinear_ref(x, Hi, Wi, Ho, Wo, mutant=mut), ref, bound), (mut, dt)


@pytest.mark.parametrize("h,w", [(9, 17), (17, 33), (33, 9)])
def test_region_probe_is_exact_and_rejects_mutants(h, w):
    tokens, pts, img = rp.region_probe(3, h, w, 8, 5, 256, _gen(5))
    assert sorted(img.tolist()) != img.tolist()
    ref = rp.region_ref(tokens, h, w, pts, img)
    assert _exact(ref, torch.float32)
    for dt in DT16:
        for mut in rp.REGION_MUTANTS:
            assert _differs(rp.stored(rp.region_ref(tokens, h, w, pts, img, mut), dt), rp.stored(ref, dt)), (mut, dt)


# ---------------------------------------------------------------------------------------------------------------
# task heads
# ---------------------------------------------------------------------------------------------------------------
HEADS_CASES = [  # Q, H4, W4, ratio, ncls, K; the first six are the geometries tests/test_resample_probes_gpu.py runs
    (37, 12, 10, 4, 47, 100),
    (104, 8, 6, 8, 133, 256),
    (100, 20, 18, 4, 48, 256),
    (112, 3, 22, 8, 144, 1),
    (1, 12, 10, 4, 1, 1),
    (100, 21, 17, 4, 134, 257),
    (104, 8, 6, 8, 133, 257),
    (100, 20, 18, 2, 48, 256),
    (112, 9, 22, 1, 144, 1),
]


@pytest.mark.parametrize("Q,H4,W4,ratio,ncls,K", HEADS_CASES)
def test_heads_probe_is_exact_and_rejects_mutants(Q, H4, W4, ratio, ncls, K):
    logits, probsT, wq, negq, slots = rp.heads_probe(Q, H4, W4, ratio, ncls, K)
    H, W = H4 * ratio, W4 * ratio
    x = rp.heads_x(logits, H, W)
    assert torch.equal(x * 256, torch.round(x * 256)) and x.abs().max() <= 127
    ref = rp.heads_ref(x, probsT, wq, negq, slots, ncls)
    props = rp.probe_properties(x, ref, Q)
    assert props["decided"]                                             # every pixel decided or an exact tie
    assert ref["stats"][:, 0].ne(ref["stats"][:, 2]).any()
    assert props["zero_rows"] and props["zero_free_rows"]               # zeros in some warp rows, not in others
    assert props["tie_wins"] or Q <= 11                                 # the lower-index tie-break is observable
    for a, b in rp.TIE_PAIRS:
        if b < Q:
            assert torch.equal(x[a], x[b]) and wq[a] == wq[b]
    exact = ("ids", "in_mask", "inst")
    for mut in rp.HEADS_MUTANTS:
        m = rp.heads_ref(rp.heads_x(logits, H, W, mutant=mut if mut == "tap_shift" else None),
                         probsT, wq, negq, slots, ncls, mutant=mut)
        hit = any(_differs(torch.nan_to_num(m[k], nan=-7.0), torch.nan_to_num(ref[k], nan=-7.0)) for k in exact)
        hit = hit or _differs(m["stats"][:, [0, 2, 3, 4]], ref["stats"][:, [0, 2, 3, 4]])
        hit = hit or _missed(m["sem"], ref["sem"], ref["sem_bound"])
        if (mut == "tie_high" and Q <= 11) or (mut == "slot_reverse" and K == 1):
            continue
        assert hit, mut
    # the float64 outputs alone reject the mutants that touch them
    for mut in ("sem_class_shift", "sem_pixel_shift", "drop_last_ctile", "drop_last_qtile"):
        m = rp.heads_ref(x, probsT, wq, negq, slots, ncls, mutant=mut)
        assert _missed(m["sem"], ref["sem"], ref["sem_bound"]), mut
    m = rp.heads_ref(x, probsT, wq, negq, slots, ncls, mutant="gt_ge_swap")
    assert _differs(m["stats"][:, 0], ref["stats"][:, 0]) and _differs(m["stats"][:, 2], ref["stats"][:, 2])


def test_heads_composed_probe_is_exact():
    Q, H4, W4 = 37, 10, 12
    logits, probsT, wq, negq, slots = rp.heads_probe(Q, H4, W4, 4, 47, 100)
    crop = (40, 48, 36, 40)                       # Hp = 4 H4, crop, then x2 (oh / H = 1/2)
    x = rp.heads_x(logits, 72, 80, crop)
    assert torch.equal(x * 4096, torch.round(x * 4096))
    ref = rp.heads_ref(x, probsT, wq, negq, slots, 47)
    assert bool(ref["ids_clear"].all())
    m = rp.heads_ref(rp.heads_x(logits, 72, 80, crop, mutant="tap_shift"), probsT, wq, negq, slots, 47)
    assert _differs(m["inst"].nan_to_num(-7.0), ref["inst"].nan_to_num(-7.0))


def test_sigmoid_sum_bound_rejects_a_lost_tile_row():
    """The fast kernel's bound on sum(sigma [x > 0]) at 256^2 (264 CTA partials) is 10x below what a lost 16-pixel
    tile row of the query's average positive pixel removes."""
    logits, probsT, wq, negq, slots = rp.heads_probe(100, 64, 64, 4, 134, 100, zeros=False)
    ref = rp.heads_ref(rp.heads_x(logits, 256, 256), None, None, None, None, 0, rows=264)
    n, tot = ref["stats"][:, 0], ref["stats"][:, 1]
    assert (n > 0).all() and (ref["sig_bound_fast"] * 10 < 16 * tot / n).all()


# ---------------------------------------------------------------------------------------------------------------
# the fast kernel's fixed-point sum
# ---------------------------------------------------------------------------------------------------------------
def test_fixed_point_payload_and_carry():
    assert rp.fixed_point_payload(1.0) == 1 << 22 and rp.fixed_point_payload(0.0) == 0
    assert rp.fixed_point_payload(0.5) == 1 << 21
    sat = [(1 << 22, 1 << 22)] * 255                                  # 255 tiles of saturated pixels: 2^23 per add
    assert rp.fixed_point_total(sat) == 255 << 23
    mixed = [(rp.fixed_point_payload(0.5 + i / 1024), rp.fixed_point_payload(0.75) if i % 3 else 0) for i in range(255)]
    want = sum(a + b for a, b in mixed)
    assert rp.fixed_point_total(mixed) == want
    wrong = {"carry of it - 1 tiles": lambda it: ((it - 1) << 31) & 0xFFFFFFFF,
             "carry 2^30 per tile": lambda it: (it << 30) & 0xFFFFFFFF,
             "no carry": lambda it: 0}
    for name, carry in wrong.items():
        # an odd tile count exposes every wrong carry in the saturated and the mixed sums
        for case, w in ((sat, 255 << 23), (mixed, want), (sat[:37], 37 << 23)):
            assert rp.fixed_point_total(case, carry) != w, name
    # past 511 tiles a slot's payload (<= 2^23 per tile) would wrap: the 255-tile limit keeps it below 2^31
    assert 255 * (1 << 23) < 1 << 31


def test_fast_max_tiles_geometry():
    for sms in (132, 114, 78):
        H4, W4, H, W = rp.fast_max_tiles_geometry(sms)
        tiles = (H // 8) * (W // 16)
        ctas = min(tiles, 2 * sms)
        assert -(-tiles // ctas) == 255 and W4 % 2 == 0 and H == 8 * H4 and W == 8 * W4


CROP_GEOMETRIES = {  # H4, W4, Hp, Wp, oh, ow, H, W: tests/test_postprocess.py's composed crop geometries
    "down": (64, 64, 256, 256, 192, 256, 120, 160),
    "up": (48, 64, 192, 256, 150, 200, 300, 400),
    "portrait": (64, 64, 256, 256, 256, 171, 640, 427),
    "coco-1024": (256, 256, 1024, 1024, 768, 1024, 480, 640),
}
CROP_MUTANTS = ("tie_high", "last_tile_row", "last_tile_col", "tap_shift", "sem_class_shift", "sem_pixel_shift",
                "drop_last_qtile", "drop_last_ctile", "slot_reverse")


@pytest.mark.parametrize("geom", ["down", "up", "portrait"])
def test_crop_float64_probe_misses_mutants_by_10x(geom):
    """The composed-crop bound of tests/test_resample_probes_gpu.py, widened 10x (bx, sem and sum(sigma) bounds), still
    rejects every mutant; the reference itself passes at 1x.  Q = 37 keeps the float64 maps small (coco-1024 runs on
    the GPU only, with the same check)."""
    H4, W4, Hp, Wp, oh, ow, H, W = CROP_GEOMETRIES[geom]
    Q, ncls, K = 37, 47, 100
    crop = (Hp, Wp, oh, ow)
    logits, probsT, wq, negq, slots = rp.heads_probe(Q, H4, W4, 4, ncls, K)
    bx = rp.crop_x_bound(logits, crop, H, W)
    assert bx < 0.05
    x = rp.heads_x(logits, H, W, crop)
    rows = ((W + 15) // 16) * ((H + 7) // 8)
    ref = rp.heads_ref(x, probsT, wq, negq, slots, ncls, rows=rows)
    assert rp.crop_violations(ref, ref, probsT, ncls, slots, bx) == []
    assert (x.abs() <= bx).float().mean() < 1e-3                       # few pixels may flip
    for mut in CROP_MUTANTS:
        xm = rp.heads_x(logits, H, W, crop, mutant="tap_shift") if mut == "tap_shift" else x
        m = rp.heads_ref(xm, probsT, wq, negq, slots, ncls, mutant=mut, rows=rows)
        assert rp.crop_violations(m, ref, probsT, ncls, slots, bx, scale=10), mut
