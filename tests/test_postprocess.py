"""Task heads: the fused post-processing (one kernel on the low-resolution logits) equals the step-by-step
path that mirrors the reference (llava_phi.py:308-447) on the up-sampled map.
CPU: python glue with the kernel emulated (tests/emu.py); GPU: the real kernel."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import emu
from psalm_b200 import postprocess as PP


def _inputs(seed, Q=100, H4=24, W4=40, ncls=20, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    logits = (torch.randn(Q, H4, W4, generator=g) * 4).to(dtype)
    cls = torch.randn(Q, ncls + 1, generator=g) * 4
    cls[:30, : ncls] += 6 * F.one_hot(torch.randint(0, ncls, (30,), generator=g), ncls)   # confident queries
    seg = torch.randn(Q, 1, generator=g)
    thing = [True] * (ncls // 2) + [False] * (ncls - ncls // 2)
    return logits, cls, seg, thing


def _reference_path(logits, cls, seg, thing, H, W, task):
    mp = F.interpolate(logits.float()[None], size=(H, W), mode="bilinear", align_corners=False)[0]
    r = {}
    if task in ("semantic", "panoptic"):
        r["sem_seg"] = PP.semantic_inference(cls, mp)
    if task in ("instance", "panoptic"):
        r["instances"] = PP.instance_inference(cls, mp, 100, thing, task == "panoptic")
    if task == "panoptic":
        r["panoptic_seg"] = PP.panoptic_inference(cls, mp, thing)
    if task == "referring":
        r["instances"] = PP.seg_instance_inference(seg, mp, 100)
    return r


def _fused(kernels, logits, cls, seg, thing, H, W, task):
    """The fused task heads of one image: fused_device_batch on a batch of one, then fused_host."""
    (d,) = PP.fused_device_batch(kernels, logits[None], [(H, W)], None if task == "referring" else cls[None],
                                 seg[None] if task == "referring" else None,
                                 PP.thing_tensor(thing, logits.device) if task == "panoptic" else None,
                                 task in ("semantic", "panoptic"), task in ("instance", "panoptic"), task == "panoptic",
                                 task == "referring", 100, 0.8)
    return PP.fused_host(d, thing, 0.8)


def _compare(ref, got, task, sem_tol):
    if "sem_seg" in ref:
        err = (got["sem_seg"].float().cpu() - ref["sem_seg"].cpu()).abs().max() / ref["sem_seg"].abs().max()
        assert err < sem_tol, err
    if "panoptic_seg" in ref:
        pr, ir = ref["panoptic_seg"]
        pg, ig = got["panoptic_seg"]
        assert ir == ig
        assert (pr.cpu() != pg.cpu()).float().mean() < 1e-3
    if "instances" in ref:
        a, b = ref["instances"], got["instances"]
        assert len(a.scores) == len(b.scores)
        key = lambda inst: sorted(zip(inst.query_index.cpu().tolist(),  # noqa: E731
                                      (inst.pred_classes.cpu().tolist() if inst.has("pred_classes") else [0] * len(inst.scores)),
                                      range(len(inst.scores))))
        ka, kb = key(a), key(b)
        assert [k[:2] for k in ka] == [k[:2] for k in kb]
        ia, ib = [k[2] for k in ka], [k[2] for k in kb]
        assert torch.allclose(a.scores.cpu()[ia], b.scores.cpu()[ib], rtol=2e-3, atol=1e-5)
        assert (a.pred_masks.cpu()[ia] != b.pred_masks.cpu()[ib]).float().mean() < 1e-4


@pytest.mark.parametrize("task", ["panoptic", "instance", "semantic", "referring"])
def test_fused_heads_batch_of_one_cpu(monkeypatch, task):
    from psalm_b200 import kernels
    monkeypatch.setattr(kernels, "postproc_fused", emu.postproc_fused)
    logits, cls, seg, thing = _inputs(3)
    H, W = 96, 160
    ref = _reference_path(logits, cls, seg, thing, H, W, task)
    got = _fused(kernels, logits, cls, seg, thing, H, W, task)
    _compare(ref, got, task, 2e-3)


@pytest.mark.parametrize("task", ["panoptic", "instance", "semantic", "referring"])
def test_batched_glue_cpu(monkeypatch, task):
    """fused_device_batch (the small algebra of all images of a step in one set of launches) gives, image by image,
    what the step-by-step reference path gives - three images with different logits / class scores."""
    from psalm_b200 import kernels
    monkeypatch.setattr(kernels, "postproc_fused", emu.postproc_fused)
    H, W = 96, 160
    per = [_inputs(10 + b) for b in range(3)]
    thing = per[0][3]
    logits = torch.stack([p[0] for p in per])
    cls = None if task == "referring" else torch.stack([p[1] for p in per])
    seg = torch.stack([p[2] for p in per]) if task == "referring" else None
    ds = PP.fused_device_batch(kernels, logits, [(H, W)] * 3, cls, seg, PP.thing_tensor(thing, "cpu") if task == "panoptic" else None,
                               task in ("semantic", "panoptic"), task in ("instance", "panoptic"), task == "panoptic",
                               task == "referring", 100, 0.8)
    assert len(ds) == 3
    for b in range(3):
        got = PP.fused_host(ds[b], thing, 0.8)
        ref = _reference_path(per[b][0], per[b][1], per[b][2], thing, H, W, task)
        _compare(ref, got, task, 2e-3)


@pytest.mark.gpu
@pytest.mark.parametrize("task", ["panoptic", "instance", "semantic", "referring"])
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("shape", [(24, 40, 96, 160), (50, 66, 200, 264), (13, 21, 61, 85)])
def test_fused_heads_batch_of_one_gpu(task, dt, shape):
    from psalm_b200 import kernels
    H4, W4, H, W = shape
    logits, cls, seg, thing = _inputs(5, H4=H4, W4=W4, dtype=dt)
    ref = _reference_path(logits.float(), cls, seg, thing, H, W, task)
    got = _fused(kernels, logits.cuda(), cls.cuda(), seg.cuda(), thing, H, W, task)
    _compare(ref, got, task, 3e-3)


def _set_impl(impl):
    from psalm_b200 import _lib
    _lib.check(_lib.lib().psalm_set_postproc_impl(impl), "psalm_set_postproc_impl")


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("shape", [(24, 40, 96, 160), (50, 66, 200, 264), (25, 34, 100, 136), (12, 20, 96, 160),
                                   (64, 64, 256, 256)])
@pytest.mark.parametrize("Q,ncls", [(100, 133), (37, 20), (112, 144)])
def test_tensor_core_kernel_vs_generic_gpu(dt, shape, Q, ncls):
    """The tensor-core formulation (csrc/postproc_fast.cu) against the torch restatement of the op and against the
    generic kernel: exact integer outputs (counts, ids, instance masks) away from fp ties, fp sums to 1e-5."""
    from psalm_b200 import kernels
    H4, W4, H, W = shape
    g = torch.Generator().manual_seed(11)
    logits = (torch.randn(Q, H4, W4, generator=g) * 4).to(dt)
    logits[:, ::5, ::3] = 0          # exact zeros: (x >= 0) differs from (x > 0)
    logits[3] = 0
    probs = F.softmax(torch.randn(Q, ncls + 1, generator=g) * 3, -1)[:, :-1]
    probsT = torch.zeros(144, 112, dtype=torch.float16)
    probsT[:ncls, :Q] = probs.t().half()
    keep = torch.rand(Q, generator=g) > 0.5
    wq = torch.where(keep, torch.rand(Q, generator=g), torch.zeros(Q))
    negq = keep.float() - 1
    slots = torch.randint(-1, Q, (100,), generator=g).to(torch.int32)
    ref = emu.postproc_fused(logits, H, W, probsT, wq, negq, slots, ncls)
    outs = {}
    try:
        for impl in (1, 2):
            if impl == 1 and Q > 104:
                continue
            _set_impl(impl)
            outs[impl] = kernels.postproc_fused(logits.cuda(), H, W, probsT.cuda(), wq.cuda(), negq.cuda(), slots.cuda(), ncls)
            again = kernels.postproc_fused(logits.cuda(), H, W, probsT.cuda(), wq.cuda(), negq.cuda(), slots.cuda(), ncls)
            for k in ("sem_seg", "ids", "in_mask", "stats"):
                assert torch.equal(outs[impl][k], again[k]), (impl, k)      # run-to-run deterministic
    finally:
        _set_impl(0)
    x = F.interpolate(logits.float()[None], size=(H, W), mode="bilinear", align_corners=False)[0]
    for impl, o in outs.items():
        st = o["stats"].cpu()
        # counts: the blend is exact up to fp32 summation order, so only |x| ~ 1e-7 pixels may flip
        near = (x.abs() < 1e-5) & (x != 0)
        slack = near.flatten(1).sum(1).float()
        assert ((st[:, 0] - ref["stats"][:, 0]).abs() <= slack).all(), impl
        assert ((st[:, 2] - ref["stats"][:, 2]).abs() <= slack).all(), impl
        assert torch.allclose(st[:, 1], ref["stats"][:, 1], rtol=1e-3 if impl == 1 else 2e-5, atol=1e-2), impl
        sem_err = (o["sem_seg"].cpu() - ref["sem_seg"]).abs().max() / ref["sem_seg"].abs().max()
        assert sem_err < 2e-3, (impl, sem_err)
        mism = (o["ids"].cpu() != ref["ids"]).float().mean()
        assert mism < 1e-4, (impl, mism)
        same = o["ids"].cpu() == ref["ids"]
        assert ((o["in_mask"].cpu() != ref["in_mask"]) & same & ~near.any(0)).sum() == 0, impl
        assert torch.equal(st[:, 3].sum(), torch.tensor(float(H * W))), impl
        valid = slots >= 0
        bad = (o["inst_masks"].cpu()[valid] != ref["inst_masks"][valid]).flatten(1).sum(1).float()
        assert (bad <= slack[slots[valid].long()]).all(), impl
    if 1 in outs and 2 in outs:
        assert torch.equal(outs[1]["ids"], outs[2]["ids"]) or (outs[1]["ids"] != outs[2]["ids"]).float().mean() < 1e-5
        assert torch.allclose(outs[1]["stats"][:, [0, 2]], outs[2]["stats"][:, [0, 2]], atol=2)


@pytest.mark.gpu
def test_tensor_core_path_forced_unsupported_raises():
    from psalm_b200 import kernels, _lib
    logits = torch.randn(10, 13, 21, device="cuda")      # fp32: tensor-core path unsupported
    try:
        _set_impl(2)
        with pytest.raises(_lib.PsalmKernelError):
            kernels.postproc_fused(logits, 61, 85)
    finally:
        _set_impl(0)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float32], ids=["bf16", "f32"])
@pytest.mark.parametrize("geom", [(64, 64, 256, 256, 192, 256, 120, 160), (48, 64, 192, 256, 150, 200, 300, 400),
                                  (64, 64, 256, 256, 256, 171, 640, 427), (40, 40, 160, 160, 160, 160, 160, 160),
                                  (256, 256, 1024, 1024, 768, 1024, 480, 640)],
                         ids=["down", "up", "portrait", "identity", "coco-1024"])
def test_composed_crop_resize_kernel(dt, geom):
    """The reference's eval flow - up-sample to the padded size, crop to the un-padded box, resize to the original size
    (sem_seg_postprocess inside eval_seg, llava_phi.py:1399-1430) - composed inside the fused kernel, against the torch
    restatement that materialises both intermediates."""
    from psalm_b200 import kernels
    H4, W4, Hp, Wp, oh, ow, H, W = geom
    Q, ncls = 100, 133
    g = torch.Generator().manual_seed(5)
    logits = (torch.randn(Q, H4, W4, generator=g) * 4).to(dt)
    probs = F.softmax(torch.randn(Q, ncls + 1, generator=g) * 3, -1)[:, :-1]
    probsT = torch.zeros(144, 112, dtype=torch.float16)
    probsT[:ncls, :Q] = probs.t().half()
    keep = torch.rand(Q, generator=g) > 0.5
    wq = torch.where(keep, torch.rand(Q, generator=g), torch.zeros(Q))
    negq = keep.float() - 1
    slots = torch.randint(-1, Q, (100,), generator=g).to(torch.int32)
    assert kernels.postproc_crop_supported(Q, H4, W4, Hp, Wp, oh, ow, H, W, ncls)
    ref = emu.postproc_fused(logits, H, W, probsT, wq, negq, slots, ncls, crop=(Hp, Wp, oh, ow))
    o = kernels.postproc_fused(logits.cuda(), H, W, probsT.cuda(), wq.cuda(), negq.cuda(), slots.cuda(), ncls, crop=(Hp, Wp, oh, ow))
    torch.cuda.synchronize()
    x = F.interpolate(F.interpolate(logits.float()[None], size=(Hp, Wp), mode="bilinear", align_corners=False)[:, :, :oh, :ow],
                      size=(H, W), mode="bilinear", align_corners=False)[0]
    near = (x.abs() < 1e-4)
    slack = near.flatten(1).sum(1).float()
    st = o["stats"].cpu()
    assert ((st[:, 0] - ref["stats"][:, 0]).abs() <= slack).all()
    assert ((st[:, 2] - ref["stats"][:, 2]).abs() <= slack).all()
    assert torch.allclose(st[:, 1], ref["stats"][:, 1], rtol=2e-3, atol=5e-2)
    assert (o["sem_seg"].cpu() - ref["sem_seg"]).abs().max() / ref["sem_seg"].abs().max() < 2e-3
    assert (o["ids"].cpu() != ref["ids"]).float().mean() < 2e-4
    assert torch.equal(st[:, 3].sum(), torch.tensor(float(H * W)))
    valid = slots >= 0
    bad = (o["inst_masks"].cpu()[valid] != ref["inst_masks"][valid]).flatten(1).sum(1).float()
    assert (bad <= slack[slots[valid].long()]).all()
