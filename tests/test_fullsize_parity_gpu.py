"""Full-size parity of the BENCHMARKED path against the CPU oracle (BASELINE.json configs C1-C5 at their real
sizes, Swin-B + Phi-1.5).  One oracle pass per configuration (10-25 s on the GPU box's host cores); the oracle
gets the bf16-rounded weights, and both GPU runs are built from exactly those values:

  * fp32 storage (SIMT kernels, library sgemm, exact task heads): north_star's "1e-3 rel on mask logits,
    bit-exact argmax class ids" — asserted at full size;
  * bf16 storage through the CUDA-graph path that bench.py times (window_mma / causal flash / cross-attention /
    MSDeformAttn / mask projection / postproc_fast / wgmma linear layers): weights are identical to the oracle's, so
    the residual is activation storage rounding + kernel error.  Asserted tolerances are fixed bounds (the value
    observed on the GPU is recorded beside each bound), plus per-stage errors, free-running and teacher-forced, the masked decoder
    layer by layer on the oracle's states and masks, and the oracle's own sensitivity to bf16 input rounding
    (oracle/parity.py): the decoder thresholds mask logits into attention masks, a discontinuity the reference has too.
"""
import json
import os

import pytest
import torch

from psalm_b200 import synth
from psalm_b200.layout import PsalmConfig

pytestmark = pytest.mark.gpu

# (task, H, W, n_classes) per BASELINE.json configuration
CONFIGS = {
    "C1_panoptic_640": ("panoptic", 640, 640, 134),
    "C2_panoptic_1024": ("panoptic", 1024, 1024, 134),
    "C3_referring_1024": ("referring", 1024, 1024, 0),
    "C4_instance_1024": ("instance", 1024, 1024, 81),
    "C5_semantic_ade150_1333": ("semantic", 1333, 1333, 151),
}
# bf16 bounds: (mask-logit l2-rel, mask-logit max-rel, class / SEG-logit max-rel, min mask-sign agreement); the trailing
# comment holds the values observed on an H100 (l2 / max / class / sign).  The class ARG-MAX is
# not bounded for bf16: with random weights the 134 class logits of a query are near ties (C1: 53 % agreement at a
# class-logit error of 5.7 %), it is asserted exactly on the fp32 path.
BF16_BOUNDS = {
    "C1_panoptic_640": (0.076, 0.146, 0.115, 0.980),          # 0.0400 / 0.0733 / 0.0667 / 0.9896
    "C2_panoptic_1024": (0.040, 0.058, 0.079, 0.989),         # 0.0204 / 0.0251 / 0.0407 / 0.9943
    "C3_referring_1024": (0.039, 0.050, 0.061, 0.989),        # 0.0201 / 0.0252 / 0.0210 / 0.9943
    "C4_instance_1024": (0.035, 0.052, 0.074, 0.990),         # 0.0198 / 0.0264 / 0.0276 / 0.9946
    "C5_semantic_ade150_1333": (0.080, 0.173, 0.129, 0.979),  # 0.0390 / 0.0751 / 0.0705 / 0.9902
}
# teacher-forced bounds (every stage / every decoder layer fed the oracle's inputs): observed <= 1.0e-2 for the stages
# up to the pixel decoder, so 2e-2; decoder layers: see LAYER_BOUND
STAGE_BOUND = 2e-2
LAYER_BOUND = 2e-2
REPORT = os.environ.get("PSALM_PARITY_REPORT")     # optional JSON file collecting the measured errors


@pytest.fixture(scope="module")
def weights():
    from oracle import parity
    cfg = PsalmConfig()
    sd = synth.synth_state_dict(cfg, seed=0)
    return cfg, parity.round_sd(sd, torch.bfloat16)


def _oracle(sd, inp, task):
    from oracle import psalm_oracle as O
    torch.set_num_threads(min(32, os.cpu_count()))
    with torch.no_grad():
        return O.eval_seg(sd, inp["input_ids"], inp["attention_mask"], inp["images"], inp["seg_info"],
                          class_name_ids=inp.get("class_name_ids"), cls_indices=inp.get("cls_indices"),
                          class_name_embedding_indices=inp.get("class_name_embedding_indices"),
                          token_refer_id=inp.get("token_refer_id"),
                          refer_embedding_indices=inp.get("refer_embedding_indices"),
                          is_thing_list=inp.get("is_thing_list"), task=task, return_intermediates=True)


def _gpu(model, inp, H, W):
    kw = {k: inp[k] for k in ("class_name_ids", "cls_indices", "class_name_embedding_indices", "token_refer_id",
                              "refer_embedding_indices", "is_thing_list") if k in inp}
    plan = model.make_plan(inp["input_ids"], inp["attention_mask"], (H, W), inp.get("class_name_ids"),
                           inp.get("cls_indices"), inp.get("class_name_embedding_indices"), inp.get("token_refer_id"),
                           inp.get("refer_embedding_indices")).to("cuda")
    trace = {}
    out = model.forward_core(inp["images"].cuda(), plan, trace=trace)
    res = model.eval_seg(input_ids=inp["input_ids"], attention_mask=inp["attention_mask"], images=inp["images"],
                         seg_info=inp["seg_info"], **kw)
    torch.cuda.synchronize()
    return out, trace, res


@pytest.mark.parametrize("name", list(CONFIGS))
def test_full_size_vs_oracle(weights, name):
    from oracle import parity
    from psalm_b200.psalm import PSALM
    cfg, sd = weights
    task, H, W, ncls = CONFIGS[name]
    inp = synth.synth_inputs(batch=1, height=H, width=W, task=task, n_classes=ncls, seed=1)
    if task != "panoptic":
        inp.pop("is_thing_list", None)
    ores, it = _oracle(sd, inp, task)
    report = {"config": name}

    # ---- fp32 storage: the north-star tolerance, at full size
    m32 = PSALM(sd, cfg, torch.float32, "cuda", task)
    out, trace, res = _gpu(m32, inp, H, W)
    f32 = dict(parity.final_metrics(out, it), **parity.result_metrics(res, ores, task))
    print("\n[%s] fp32: %s" % (name, parity.fmt(f32)))
    report["fp32"] = f32
    del m32, out, trace, res
    torch.cuda.empty_cache()

    # ---- bf16 storage through the graph path the bench times
    mb = PSALM(sd, cfg, torch.bfloat16, "cuda", task, use_cuda_graph=True)
    out, trace, res = _gpu(mb, inp, H, W)
    b16 = dict(parity.final_metrics(out, it), **parity.result_metrics(res, ores, task))
    free = parity.free_stage_errors(trace, it)
    forced = parity.forced_stage_errors(mb, it, inp["images"])
    layers = parity.forced_layer_errors(mb, it)
    sens = parity.predictor_sensitivity(sd, it, torch.bfloat16)
    print("[%s] bf16: %s" % (name, parity.fmt(b16)))
    print("[%s] bf16 free-running stage l2-rel : %s" % (name, parity.fmt(free)))
    print("[%s] bf16 teacher-forced stage l2-rel: %s" % (name, parity.fmt(forced)))
    print("[%s] bf16 decoder, layer-wise teacher-forced: %s" % (name, parity.fmt(layers)))
    print("[%s] ORACLE decoder re-run on bf16-rounded inputs (conditioning of the reference itself): %s" % (name, parity.fmt(sens)))
    report.update(bf16=b16, bf16_free_stage_l2rel=free, bf16_forced_stage_l2rel=forced, bf16_decoder_layers_forced=layers,
                  oracle_decoder_sensitivity_to_bf16_inputs=sens)
    if REPORT:
        allr = json.load(open(REPORT)) if os.path.exists(REPORT) else {}
        allr[name] = report
        json.dump(allr, open(REPORT, "w"), indent=1)

    assert f32["mask_logit_maxrel"] < 1e-3
    if "class_argmax_agree" in f32:
        assert f32["class_argmax_agree"] == 1.0
    if "seg_top1_agree" in f32:
        assert f32["seg_top1_agree"] == 1.0
    if "panoptic_pixel_agree" in f32:
        assert f32["panoptic_pixel_agree"] > 0.998 and f32["panoptic_segments_equal"] == 1.0
    if "sem_argmax_agree" in f32:
        assert f32["sem_argmax_agree"] > 0.998
    l2, mx, clsmx, sign = BF16_BOUNDS[name]
    assert b16["mask_logit_l2rel"] < l2 and b16["mask_logit_maxrel"] < mx and b16["mask_sign_agree"] >= sign
    assert b16.get("class_logit_maxrel", b16.get("seg_logit_maxrel", 0.0)) < clsmx
    # kernels + storage rounding of each stage in isolation (no inherited error, no mask-threshold chaos)
    for k in ("swin_res2", "swin_res3", "swin_res4", "swin_res5", "img_tok", "hidden", "mask_features", "ms0", "ms1", "ms2"):
        assert forced[k] < STAGE_BOUND, (k, forced[k])
    assert layers["layer_l2rel_max"] < LAYER_BOUND, layers
    assert layers["mask_bit_agree_off_threshold_min"] > 0.9995, layers   # bits whose oracle logit is > 5 % of the rms away from 0
