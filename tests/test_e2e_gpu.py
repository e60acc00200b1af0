"""End-to-end parity of psalm_b200.PSALM (CUDA kernels through the C ABI) against the fixtures the
UNMODIFIED reference produced (tests/golden/e2e_*.npz) and against the oracle, on the GPU.

Tolerances.  north_star: "within 1e-3 rel on mask logits, bit-exact argmax class ids".  We measure
rel = max|err| / max|ref| on the final mask logits:
  fp32 run   : < 1e-3   (asserted; typically ~1e-5) and class argmax exactly equal
  fp16 / bf16: storage rounding accumulates over ~60 layers; the l2-relative error is asserted
               (< 4e-2 fp16, < 2.5e-1 bf16) with the observed values printed (DESIGN.md "precision"),
               class-argmax agreement >= 97 % / 90 %."""
import numpy as np
import pytest
import torch

from psalm_b200 import synth
from psalm_b200.layout import PhiConfig, PsalmConfig

pytestmark = pytest.mark.gpu
SMALL = PsalmConfig(phi=PhiConfig(hidden=256, layers=2, heads=4, inter=1024))
CASES = [("panoptic", 192, 192, 20, 0, 1, False), ("panoptic", 200, 264, 12, 3, 1, False),
         ("referring", 192, 192, 0, 5, 1, False), ("panoptic", 96, 128, 7, 7, 2, True)]


def _run(case, dtype):
    from psalm_b200.psalm import PSALM
    task, H, W, ncls, seed, batch, ragged = case
    sd = synth.synth_state_dict(SMALL, seed=seed)
    inp = synth.synth_inputs(batch=batch, height=H, width=W, task=task, n_classes=ncls, seed=seed + 1, ragged=ragged)
    m = PSALM(sd, SMALL, dtype, "cuda", task)
    plan = m.make_plan(inp["input_ids"], inp["attention_mask"], (H, W), inp.get("class_name_ids"), inp.get("cls_indices"),
                       inp.get("class_name_embedding_indices"), inp.get("token_refer_id"),
                       inp.get("refer_embedding_indices")).to("cuda")
    out = m.forward_core(inp["images"].cuda(), plan)
    kw = {k: inp[k] for k in ("class_name_ids", "cls_indices", "class_name_embedding_indices", "token_refer_id",
                              "refer_embedding_indices", "is_thing_list") if k in inp}
    res = m.eval_seg(input_ids=inp["input_ids"], attention_mask=inp["attention_mask"], images=inp["images"],
                     seg_info=inp["seg_info"], **kw)
    torch.cuda.synchronize()
    return out, res


@pytest.mark.parametrize("case", CASES, ids=lambda c: "%s_%dx%d_b%d" % (c[0], c[1], c[2], c[5]))
def test_fp32_matches_reference_golden(golden, case):
    task, H, W, ncls, seed, batch, ragged = case
    g = golden("e2e_%s_%dx%d_b%d.npz" % (task, H, W, batch))
    out, res = _run(case, torch.float32)
    pm = out["pred_masks"].float().cpu().reshape(-1)[torch.from_numpy(g["pred_masks_idx"])].numpy()
    rel = np.abs(pm - g["pred_masks"]).max() / np.abs(g["pred_masks"]).max()
    print("fp32 mask-logit rel err %.3e" % rel)
    assert rel < 1e-3
    if "pred_class_name_logits" in g:
        cl = out["pred_class_name_logits"].float().cpu().numpy()
        assert np.array_equal(cl.argmax(-1), g["pred_class_name_logits"].argmax(-1))
        assert np.allclose(cl, g["pred_class_name_logits"], rtol=1e-3, atol=2e-3)
    if "pred_SEG_logits" in g:
        assert np.allclose(out["pred_SEG_logits"].float().cpu().numpy(), g["pred_SEG_logits"], rtol=1e-3, atol=2e-3)
    if "panoptic_seg" in g:
        pan, info = res[0]["panoptic_seg"]
        assert (pan.cpu().numpy() != g["panoptic_seg"]).mean() < 2e-3
        assert [[d["id"], int(d["isthing"]), d["category_id"]] for d in info] == g["panoptic_info"].tolist()
        assert (res[0]["sem_seg"].argmax(0).cpu().numpy().astype(np.uint8) != g["sem_seg_argmax"]).mean() < 2e-3
    if "inst_scores_sorted" in g:
        sc = res[0]["instances"].scores.cpu()
        order = torch.argsort(sc, descending=True, stable=True)
        assert np.allclose(sc[order].numpy(), g["inst_scores_sorted"], rtol=1e-3, atol=1e-4)
    assert len(res) == batch   # every image is post-processed (the reference stops after image 0)


@pytest.mark.parametrize("dtype,tol,agree", [(torch.float16, 4e-2, 0.97), (torch.bfloat16, 2.5e-1, 0.90)],
                         ids=["fp16", "bf16"])
def test_low_precision_tracks_reference(golden, dtype, tol, agree):
    case = CASES[0]
    g = golden("e2e_panoptic_192x192_b1.npz")
    out, res = _run(case, dtype)
    pm = out["pred_masks"].float().cpu().reshape(-1)[torch.from_numpy(g["pred_masks_idx"])].numpy()
    rel = np.abs(pm - g["pred_masks"]).max() / np.abs(g["pred_masks"]).max()
    nrm = np.linalg.norm(pm - g["pred_masks"]) / np.linalg.norm(g["pred_masks"])
    cl = out["pred_class_name_logits"].float().cpu().numpy()
    ag = (cl.argmax(-1) == g["pred_class_name_logits"].argmax(-1)).mean()
    print("%s: mask-logit max-rel %.3e, l2-rel %.3e, class-argmax agreement %.3f" % (dtype, rel, nrm, ag))
    assert np.isfinite(pm).all() and nrm < tol and ag >= agree   # tol on the l2-relative error


def test_full_size_bf16_smoke():
    """The configuration BASELINE.json's metric is quoted on: 1024^2, Swin-B + Phi-1.5, 100 queries,
    134 class names, bf16.  No oracle at this size in the GPU suite (it takes minutes on CPU):
    shapes, finiteness, run-to-run determinism and structural invariants of the outputs."""
    from psalm_b200.psalm import PSALM
    cfg = PsalmConfig()
    sd = synth.synth_state_dict(cfg, seed=0, device="cuda")
    m = PSALM(sd, cfg, torch.bfloat16, "cuda", "panoptic")
    del sd
    inp = synth.synth_inputs(batch=1, height=1024, width=1024, task="panoptic", n_classes=134, seed=1)
    kw = {k: inp[k] for k in ("class_name_ids", "cls_indices", "class_name_embedding_indices", "is_thing_list")}
    r1 = m.eval_seg(input_ids=inp["input_ids"], attention_mask=inp["attention_mask"], images=inp["images"],
                    seg_info=inp["seg_info"], **kw)
    r2 = m.eval_seg(input_ids=inp["input_ids"], attention_mask=inp["attention_mask"], images=inp["images"],
                    seg_info=inp["seg_info"], **kw)
    torch.cuda.synchronize()
    sem = r1[0]["sem_seg"]
    assert tuple(sem.shape) == (133, 1024, 1024) and torch.isfinite(sem).all()
    pan, info = r1[0]["panoptic_seg"]
    assert tuple(pan.shape) == (1024, 1024) and pan.dtype == torch.int32
    assert set(np.unique(pan.cpu().numpy()).tolist()) <= set([0] + [d["id"] for d in info])
    assert torch.equal(pan, r2[0]["panoptic_seg"][0]) and torch.equal(sem, r2[0]["sem_seg"])
    inst = r1[0]["instances"]
    assert inst.pred_masks.shape[1:] == (1024, 1024) and torch.isfinite(inst.scores).all()


def test_cuda_graph_replay_matches_eager():
    """PSALM(use_cuda_graph=True): the captured graph (network + fused task heads) gives the same results as
    eager launches, also when replayed for a second image with the same prompt structure."""
    from psalm_b200.psalm import PSALM
    task, H, W, ncls, seed, batch, ragged = ("panoptic", 192, 192, 20, 0, 1, False)
    sd = synth.synth_state_dict(SMALL, seed=seed)
    eager = PSALM(sd, SMALL, torch.bfloat16, "cuda", task, use_cuda_graph=False)
    graphed = PSALM(sd, SMALL, torch.bfloat16, "cuda", task, use_cuda_graph=True)
    for s2 in (1, 2, 1):
        inp = synth.synth_inputs(batch=batch, height=H, width=W, task=task, n_classes=ncls, seed=s2)
        kw = {k: inp[k] for k in ("class_name_ids", "cls_indices", "class_name_embedding_indices", "is_thing_list")}
        a = eager.eval_seg(input_ids=inp["input_ids"], attention_mask=inp["attention_mask"], images=inp["images"],
                           seg_info=inp["seg_info"], **kw)
        b = graphed.eval_seg(input_ids=inp["input_ids"], attention_mask=inp["attention_mask"], images=inp["images"],
                             seg_info=inp["seg_info"], **kw)
        torch.cuda.synchronize()
        assert torch.equal(a[0]["panoptic_seg"][0], b[0]["panoptic_seg"][0]) and a[0]["panoptic_seg"][1] == b[0]["panoptic_seg"][1]
        assert torch.equal(a[0]["sem_seg"], b[0]["sem_seg"])
        assert torch.allclose(a[0]["instances"].scores, b[0]["instances"].scores, rtol=1e-5, atol=1e-7)


def test_cuda_graphs_of_different_sizes_and_batches_alternate():
    """Graphs captured for several (image size, batch) keys hold device pointers of per-size cached tensors (position
    terms of the pixel decoder, K / V constants of the mask decoder): replaying A, B, C, A must keep matching eager
    launches - a cache that dropped size A's tensors when B arrived would feed the first graph freed memory."""
    from psalm_b200.psalm import PSALM
    sd = synth.synth_state_dict(SMALL, seed=0)
    eager = PSALM(sd, SMALL, torch.bfloat16, "cuda", "panoptic", use_cuda_graph=False)
    graphed = PSALM(sd, SMALL, torch.bfloat16, "cuda", "panoptic", use_cuda_graph=True)
    keys = {"A": (1, 192, 192), "B": (2, 160, 224), "C": (1, 256, 128)}
    for step, name in enumerate("ABCABA"):
        batch, H, W = keys[name]
        inp = synth.synth_inputs(batch=batch, height=H, width=W, task="panoptic", n_classes=12, seed=10 + step)
        kw = {k: inp[k] for k in ("class_name_ids", "cls_indices", "class_name_embedding_indices", "is_thing_list")}
        a = eager.eval_seg(input_ids=inp["input_ids"], attention_mask=inp["attention_mask"], images=inp["images"],
                           seg_info=inp["seg_info"], **kw)
        b = graphed.eval_seg(input_ids=inp["input_ids"], attention_mask=inp["attention_mask"], images=inp["images"],
                             seg_info=inp["seg_info"], **kw)
        torch.cuda.synchronize()
        for i in range(batch):
            assert torch.equal(a[i]["panoptic_seg"][0], b[i]["panoptic_seg"][0]), (step, name, i)
            assert torch.equal(a[i]["sem_seg"], b[i]["sem_seg"]), (step, name, i)
    assert 3 <= len(graphed._graphs) <= 6        # one graph per (size, batch, prompt length) key; none evicted


def test_cuda_graph_replays_a_prompt_whose_plan_left_the_plan_cache():
    """More referring prompts of one structure than the plan cache holds (MAX_PLANS): one forward graph serves them all,
    and replaying it for the first prompt after that prompt's cached plan was evicted and freed still gives the eager
    results - the graph reads its own copies of the plan tensors, refreshed from the live plan before each replay."""
    from psalm_b200.psalm import PSALM
    sd = synth.synth_state_dict(SMALL, seed=5)
    eager = PSALM(sd, SMALL, torch.bfloat16, "cuda", "referring", use_cuda_graph=False)
    graphed = PSALM(sd, SMALL, torch.bfloat16, "cuda", "referring", use_cuda_graph=True)
    inp = synth.synth_inputs(batch=1, height=192, width=192, task="referring", refer_len=9, seed=6)
    g = torch.Generator().manual_seed(0)
    refers = []
    for _ in range(graphed.MAX_PLANS + 2):     # same length, different refer tokens: one graph key, distinct plans
        r = inp["token_refer_id"][0].clone()
        r[:-1] = torch.randint(5, 50000, (r.numel() - 1,), generator=g)
        refers.append(r)

    def run(m, refer):
        res = m.eval_seg(input_ids=inp["input_ids"], attention_mask=inp["attention_mask"], images=inp["images"],
                         seg_info=inp["seg_info"], token_refer_id=[refer],
                         refer_embedding_indices=inp["refer_embedding_indices"])
        torch.cuda.synchronize()
        return res[0]["instances"].scores.clone(), res[0]["instances"].pred_masks.clone()
    for r in refers:
        run(graphed, r)
    assert len(graphed._graphs) == 1 and len(graphed._plans) == graphed.MAX_PLANS
    for r in (refers[0], refers[-1]):
        (a, am), (b, bm) = run(graphed, r), run(eager, r)
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-7) and torch.equal(am, bm)


def _oracle(sd, inp, task):
    from oracle import psalm_oracle as O
    phi = dict(hidden=256, layers=2, heads=4, inter=1024, eps=1e-5, theta=10000.0, rotary_frac=0.5)
    with torch.no_grad():
        return O.eval_seg(sd, inp["input_ids"], inp["attention_mask"], inp["images"], inp["seg_info"],
                          class_name_ids=inp.get("class_name_ids"), cls_indices=inp.get("cls_indices"),
                          class_name_embedding_indices=inp.get("class_name_embedding_indices"),
                          token_refer_id=inp.get("token_refer_id"),
                          refer_embedding_indices=inp.get("refer_embedding_indices"),
                          is_thing_list=inp.get("is_thing_list"), task=task, phi_cfg=phi, return_intermediates=True)


def _eval(m, inp):
    kw = {k: inp[k] for k in ("class_name_ids", "cls_indices", "class_name_embedding_indices", "token_refer_id",
                              "refer_embedding_indices", "is_thing_list") if k in inp}
    r = m.eval_seg(input_ids=inp["input_ids"], attention_mask=inp["attention_mask"], images=inp["images"],
                   seg_info=inp["seg_info"], **kw)
    torch.cuda.synchronize()
    return r


@pytest.mark.parametrize("task", ["instance", "semantic"])
def test_other_tasks_fp32_vs_oracle(task):
    """SEG_TASK instance / semantic (llava_phi.py:268-301) against the CPU oracle on the same weights."""
    from psalm_b200.psalm import PSALM
    sd = synth.synth_state_dict(SMALL, seed=11)
    inp = synth.synth_inputs(batch=1, height=160, width=224, task=task, n_classes=9, seed=12)
    inp.pop("is_thing_list", None)
    ores, it = _oracle(sd, inp, task)
    res = _eval(PSALM(sd, SMALL, torch.float32, "cuda", task), inp)
    if task == "semantic":
        a, b = res[0]["sem_seg"].cpu(), ores[0]["sem_seg"]
        assert a.shape == b.shape and (a - b).abs().max() / b.abs().max() < 1e-3
    else:
        sa = torch.sort(res[0]["instances"].scores.cpu(), descending=True).values
        sb = torch.sort(ores[0]["instances"]["scores"], descending=True).values
        assert torch.allclose(sa, sb, rtol=1e-3, atol=1e-5)
        assert res[0]["instances"].pred_masks.shape == ores[0]["instances"]["pred_masks"].shape


def test_padded_image_crop_and_resize_fp32_vs_oracle():
    """seg_info with a real padding box and an output size different from the network input: exercises the
    crop + bilinear resize of sem_seg_postprocess (llava_phi.py:1418-1430), not the fused fast path."""
    from psalm_b200.psalm import PSALM
    sd = synth.synth_state_dict(SMALL, seed=21)
    inp = synth.synth_inputs(batch=1, height=192, width=256, task="panoptic", n_classes=9, seed=22)
    pm = torch.zeros(192, 256, dtype=torch.bool)
    pm[150:, :] = True
    pm[:, 200:] = True
    inp["seg_info"] = [dict(padding_mask=pm, height=300, width=400)]
    ores, it = _oracle(sd, inp, "panoptic")
    for dtype, tol in ((torch.float32, 1e-3), (torch.bfloat16, 0.3)):
        res = _eval(PSALM(sd, SMALL, dtype, "cuda", "panoptic"), inp)
        a, b = res[0]["sem_seg"].float().cpu(), ores[0]["sem_seg"]
        assert tuple(a.shape) == tuple(b.shape) == (8, 300, 400)
        assert (a - b).norm() / b.norm() < tol
        pa, pb = res[0]["panoptic_seg"][0].cpu(), ores[0]["panoptic_seg"][0]
        assert pa.shape == pb.shape
        if dtype == torch.float32:
            assert (pa != pb).float().mean() < 2e-3 and res[0]["panoptic_seg"][1] == ores[0]["panoptic_seg"][1]


def test_fused_task_heads_track_the_oracle_bf16():
    """16-bit run with the fused task-head kernel (one image, no crop): semantic map and instance scores close
    to the fp32 oracle, panoptic segment list identical when the fp32 decision margins are not marginal."""
    from psalm_b200.psalm import PSALM
    sd = synth.synth_state_dict(SMALL, seed=0)
    inp = synth.synth_inputs(batch=1, height=192, width=192, task="panoptic", n_classes=20, seed=1)
    ores, it = _oracle(sd, inp, "panoptic")
    m = PSALM(sd, SMALL, torch.bfloat16, "cuda", "panoptic")
    assert m.fused_postprocess
    res = _eval(m, inp)
    a, b = res[0]["sem_seg"].float().cpu(), ores[0]["sem_seg"]
    assert (a - b).norm() / b.norm() < 0.2
    assert res[0]["instances"].pred_masks.shape[1:] == (192, 192)


@pytest.mark.parametrize("task,H,W,ncls,batch", [("instance", 1024, 1024, 81, 4), ("semantic", 1333, 1333, 151, 1),
                                                  ("referring", 1024, 1024, 0, 1), ("panoptic", 640, 640, 134, 2)],
                         ids=["C4_instance_b4", "C5_ade150_1333", "C3_referring", "C1_640_b2"])
def test_baseline_configs_full_size_bf16(task, H, W, ncls, batch):
    """The other BASELINE.json configurations at their real sizes (SURVEY.md section 8d: C4 COCO-instance with 81
    class names, C5 ADE-150 at 1333^2 - feature levels 168/84/42, padded to 1344, cropped back -, C3 referring,
    C1 640^2), full Swin-B + Phi-1.5 in bf16.  The CPU oracle takes minutes at these sizes, so this checks shapes,
    finiteness, run-to-run determinism and structural invariants; parity is pinned at reduced sizes above."""
    from psalm_b200.psalm import PSALM
    cfg = PsalmConfig()
    sd = synth.synth_state_dict(cfg, seed=0, device="cuda")
    m = PSALM(sd, cfg, torch.bfloat16, "cuda", task)
    del sd
    inp = synth.synth_inputs(batch=batch, height=H, width=W, task=task, n_classes=ncls, seed=3, ragged=batch > 1)
    r1, r2 = _eval(m, inp), _eval(m, inp)
    assert len(r1) == batch
    for a, b in zip(r1, r2):
        if task == "semantic":
            sem = a["sem_seg"]
            assert tuple(sem.shape) == (ncls - 1, H, W) and torch.isfinite(sem).all()
            assert float(sem.min()) >= 0.0 and torch.equal(sem, b["sem_seg"])
        if task in ("instance", "referring"):
            ia, ib = a["instances"], b["instances"]
            assert ia.pred_masks.shape[1:] == (H, W) and torch.isfinite(ia.scores).all()
            assert set(torch.unique(ia.pred_masks).tolist()) <= {0.0, 1.0}
            assert torch.equal(ia.pred_masks, ib.pred_masks) and torch.equal(ia.scores, ib.scores)
            if task == "instance":
                assert int(ia.pred_classes.max()) < ncls - 1 and len(ia.scores) == 100
        if task == "panoptic":
            pan, info = a["panoptic_seg"]
            assert tuple(pan.shape) == (H, W) and torch.equal(pan, b["panoptic_seg"][0]) and info == b["panoptic_seg"][1]
            assert set(np.unique(pan.cpu().numpy()).tolist()) <= set([0] + [d["id"] for d in info])


def test_mapper_flow_runs_the_composed_kernel_for_every_image_and_matches_the_oracle(monkeypatch):
    """The reference's real eval flow (coco_panoptic_mapper.py:148-162): image resized + padded to a square with a
    padding mask, outputs at the ORIGINAL size.  16-bit runs take the composed fused kernel (eager and CUDA graph), whose
    results must equal the step-by-step torch path on the same mask logits and track the fp32 oracle."""
    from psalm_b200 import postprocess as PP
    from psalm_b200.psalm import PSALM
    sd = synth.synth_state_dict(SMALL, seed=21)
    inp = synth.synth_inputs(batch=2, height=256, width=256, task="panoptic", n_classes=9, seed=22)
    pm = torch.zeros(256, 256, dtype=torch.bool)
    pm[192:, :] = True                       # a 4:3 image resized to 256 x 192, padded at the bottom
    inp["seg_info"] = [dict(padding_mask=pm, height=120, width=160), dict(padding_mask=pm.clone(), height=300, width=400)]
    ores, it = _oracle(sd, inp, "panoptic")
    calls = {False: [], True: []}        # per run: the crops of every fused_device_batch call
    real_b = PP.fused_device_batch

    def spy_b(*a, **k):
        calls[graph].append(k.get("crops"))
        return real_b(*a, **k)
    monkeypatch.setattr(PP, "fused_device_batch", spy_b)
    outs = {}
    for graph in (False, True):
        m = PSALM(sd, SMALL, torch.bfloat16, "cuda", "panoptic", use_cuda_graph=graph)
        m.object_mask_threshold = m.overlap_threshold = 0.0      # keep segments on random weights
        res = _eval(m, inp)
        res = _eval(m, inp)
        outs[graph] = res
        for b, (hh, ww) in enumerate(((120, 160), (300, 400))):
            assert tuple(res[b]["sem_seg"].shape) == (8, hh, ww) and tuple(res[b]["panoptic_seg"][0].shape) == (hh, ww)
            assert res[b]["instances"].pred_masks.shape[1:] == (hh, ww)
            a, o = res[b]["sem_seg"].float().cpu(), ores[b]["sem_seg"]
            assert (a - o).norm() / o.norm() < 0.2
    for graph in (False, True):     # the composed kernel ran for every image, eager and graph, never the slow path
        assert calls[graph] and all(c == [(256, 256, 192, 256)] * 2 for c in calls[graph]), (graph, calls[graph])
    for b in range(2):                                                       # graph replay == eager
        assert torch.equal(outs[False][b]["panoptic_seg"][0], outs[True][b]["panoptic_seg"][0])
        assert torch.equal(outs[False][b]["sem_seg"], outs[True][b]["sem_seg"])


def test_async_two_lane_pipeline_equals_the_blocking_call():
    """PSALM.eval_seg_async: batch k+1 submitted on the other lane before batch k is finished on a side stream (the
    pipelined loop bench.py times as e2e) must return exactly what the blocking eval_seg returns for each batch."""
    from psalm_b200.psalm import PSALM
    sd = synth.synth_state_dict(SMALL, seed=31)
    m = PSALM(sd, SMALL, torch.bfloat16, "cuda", "panoptic", use_cuda_graph=True)
    m.object_mask_threshold = m.overlap_threshold = 0.0
    batches = [synth.synth_inputs(batch=2, height=256, width=256, task="panoptic", n_classes=9, seed=40 + i) for i in range(4)]
    for inp in batches:   # one prompt structure, different images
        inp.update({k: batches[0][k] for k in batches[0] if k not in ("images", "seg_info")})
    kw = {k: batches[0][k] for k in ("class_name_ids", "cls_indices", "class_name_embedding_indices", "is_thing_list")}

    def snap(res):
        return [(r["panoptic_seg"][0].clone(), [dict(s) for s in r["panoptic_seg"][1]], r["sem_seg"].clone(),
                 r["instances"].scores.clone(), r["instances"].pred_masks.clone()) for r in res]
    want = [snap(_eval(m, inp)) for inp in batches]
    side = torch.cuda.Stream()
    got = []

    def submit(k):
        u8 = batches[k]["images"]
        return m.eval_seg_async(input_ids=batches[k]["input_ids"], attention_mask=batches[k]["attention_mask"],
                                images=m.stage_images(u8.pin_memory()), seg_info=batches[k]["seg_info"], lane=k % 2, **kw)
    pend = submit(0)
    for k in range(len(batches)):
        nxt = submit(k + 1) if k + 1 < len(batches) else None
        with torch.cuda.stream(side):
            got.append(snap(pend.result()))
        side.synchronize()
        pend = nxt
    torch.cuda.synchronize()
    for w, g in zip(want, got):
        for (wp, wi, ws, wsc, wm), (gp, gi, gs, gsc, gm) in zip(w, g):
            assert torch.equal(wp, gp) and wi == gi and torch.equal(ws, gs) and torch.equal(wsc, gsc) and torch.equal(wm, gm)
