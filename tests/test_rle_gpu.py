"""Device COCO RLE (csrc/rle.cu, psalm_b200/rle.py) against the numpy restatement of pycocotools (oracle/coco_rle.py):
byte-identical strings, round trips, area / bbox, and eval_seg(mask_format="rle") end to end."""
import numpy as np
import pytest
import torch

from oracle import coco_rle as R
from psalm_b200 import kernels, rle, synth
from psalm_b200.layout import PhiConfig, PsalmConfig

pytestmark = pytest.mark.gpu
SMALL = PsalmConfig(phi=PhiConfig(hidden=256, layers=2, heads=4, inter=1024))
SIZES = [(1, 1), (1, 37), (41, 1), (7, 33), (480, 640), (1024, 1024), (1333, 1333)]


def _patterns(H, W, seed):
    """Named uint8 [H, W] masks: empty, full, one pixel at each corner, runs that cross column boundaries, random at
    1 / 50 / 99 %, and the Fortran-order checkerboard (every run of length 1)."""
    rng = np.random.default_rng(seed)
    N = H * W
    out = {"empty": np.zeros((H, W), np.uint8), "full": np.ones((H, W), np.uint8)}
    for name, (y, x) in (("tl", (0, 0)), ("tr", (0, W - 1)), ("bl", (H - 1, 0)), ("br", (H - 1, W - 1))):
        m = np.zeros((H, W), np.uint8)
        m[y, x] = 1
        out["corner_" + name] = m
    f = np.zeros(N, np.uint8)
    for s in range(max(H // 2, 1) - 1, N, max(3 * H, 3)):     # runs of H + 2 pixels starting mid-column
        f[s:s + H + 2] = 1
    out["cross"] = f.reshape((W, H)).T.copy()
    for p in (0.01, 0.5, 0.99):
        out["rand%g" % p] = (rng.random((H, W)) < p).astype(np.uint8)
    y, x = np.mgrid[:H, :W]
    out["checker"] = ((x * H + y) % 2).astype(np.uint8)
    return out


def _as(m, dtype):
    return m.float() if dtype == torch.float32 else (m != 0 if dtype == torch.bool else m)


@pytest.mark.parametrize("H,W", SIZES, ids=["%dx%d" % s for s in SIZES])
def test_encode_is_byte_identical_to_the_oracle(H, W):
    pats = _patterns(H, W, seed=H * 7 + W)
    names = list(pats)
    want = {k: R.to_string(R.encode(v)) for k, v in pats.items()}
    counts = {k: R.encode(v) for k, v in pats.items()}
    area = {k: R.area(c) for k, c in counts.items()}
    bbox = {k: R.to_bbox(c, H, W) for k, c in counts.items()}
    base = torch.from_numpy(np.stack([pats[k] for k in names])).cuda()        # uint8 [P, H, W]
    batch = [names[i % len(names)] for i in range(100)]
    idx = torch.tensor([names.index(k) for k in batch], device="cuda")
    for dtype in (torch.float32, torch.uint8, torch.bool):
        for k, name in enumerate(names):                                       # one mask per call
            got = rle.encode(_as(base[k], dtype))
            assert got == [{"size": [H, W], "counts": want[name]}], (dtype, name)
        masks = _as(base.index_select(0, idx), dtype)                          # 100 masks in one call
        d = rle.encode_device(masks)
        dicts = rle.to_dicts(d)
        assert [x["counts"] for x in dicts] == [want[k] for k in batch], dtype
        assert all(x["size"] == [H, W] for x in dicts)
        assert d["area"].tolist() == [area[k] for k in batch]
        assert d["bbox"].tolist() == [bbox[k] for k in batch]
        if dtype == torch.uint8:
            assert torch.equal(rle.decode(d), masks)
            assert torch.equal(rle.decode(dicts[:len(names)]), base[idx[:len(names)]])
        del masks, d


def test_decode_accepts_str_counts_and_area_bbox_of_dicts():
    m = torch.from_numpy(np.stack(list(_patterns(7, 33, 0).values()))).cuda()
    enc = rle.encode(m)
    as_str = [{"size": e["size"], "counts": e["counts"].decode()} for e in enc]
    assert torch.equal(rle.decode(as_str), m)
    counts = [R.encode(x) for x in m.cpu().numpy()]
    assert rle.area(enc).tolist() == [R.area(c) for c in counts]
    assert rle.to_bbox(as_str).tolist() == [R.to_bbox(c, 7, 33) for c in counts]


def test_list_of_tensors_is_one_batch_and_empty_input_launches_nothing():
    g = torch.Generator(device="cuda").manual_seed(0)
    a = torch.rand(3, 50, 70, device="cuda", generator=g) > 0.5
    b = torch.rand(5, 50, 70, device="cuda", generator=g) > 0.9
    d = rle.encode_device([a, b])
    assert rle.to_dicts(d) == rle.encode(torch.cat([a, b]))
    before = kernels.launches()
    assert rle.encode(torch.zeros(0, 50, 70, device="cuda")) == []
    e = rle.encode_device([torch.zeros(0, 4, 4, device="cuda")])
    assert e["offsets"].tolist() == [0] and tuple(rle.decode(e).shape) == (0, 4, 4)
    assert kernels.launches() == before


def test_instances_to_coco_json_records():
    from psalm_b200.structures import Boxes, Instances
    inst = Instances((40, 30))
    g = torch.Generator(device="cuda").manual_seed(1)
    inst.pred_masks = (torch.rand(4, 40, 30, device="cuda", generator=g) > 0.7).float()
    inst.pred_boxes = Boxes(torch.zeros(4, 4))
    inst.scores = torch.tensor([0.9, 0.8, 0.7, 0.6], device="cuda")
    inst.pred_classes = torch.tensor([5, 1, 5, 2], device="cuda")
    recs = rle.instances_to_coco_json(inst, 42)
    want = R.encode_masks(inst.pred_masks.cpu().numpy())
    assert len(recs) == 4
    for r, w, c in zip(recs, want, (5, 1, 5, 2)):
        assert set(r) == {"image_id", "category_id", "bbox", "score", "segmentation"}
        assert r["image_id"] == 42 and r["category_id"] == c and r["bbox"] == [0.0, 0.0, 0.0, 0.0]
        assert isinstance(r["segmentation"]["counts"], str) and r["segmentation"]["counts"] == w["counts"].decode()
        assert r["segmentation"]["size"] == [40, 30]


def _kw(inp, mask_format=None):
    kw = {k: inp[k] for k in ("class_name_ids", "cls_indices", "class_name_embedding_indices", "token_refer_id",
                              "refer_embedding_indices", "is_thing_list") if k in inp}
    if mask_format is not None:
        kw["mask_format"] = mask_format
    return kw


def _snap(res):
    return [{k: (v.clone() if torch.is_tensor(v) else v) for k, v in r["instances"].get_fields().items()} for r in res]


@pytest.mark.parametrize("task", ["instance", "panoptic"])
@pytest.mark.parametrize("mapper", [False, True], ids=["trivial", "mapper"])
@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_eval_seg_mask_format_rle(task, mapper, graph):
    from psalm_b200.psalm import PSALM
    sd = synth.synth_state_dict(SMALL, seed=21)
    H = W = 256 if mapper else 192
    inp = synth.synth_inputs(batch=2, height=H, width=W, task=task, n_classes=9, seed=22)
    if mapper:
        pm = torch.zeros(256, 256, dtype=torch.bool)
        pm[192:, :] = True
        inp["seg_info"] = [dict(padding_mask=pm, height=120, width=160), dict(padding_mask=pm.clone(), height=300, width=400)]
    m = PSALM(sd, SMALL, torch.bfloat16, "cuda", task, use_cuda_graph=graph)
    m.object_mask_threshold = m.overlap_threshold = 0.0
    run = lambda fmt=None: m.eval_seg(input_ids=inp["input_ids"], attention_mask=inp["attention_mask"],  # noqa: E731
                                      images=inp["images"], seg_info=inp["seg_info"], **_kw(inp, fmt))
    plain = _snap(run())
    graphs = len(getattr(m, "_graphs", {}))
    dense = run("dense")
    for a, b in zip(_snap(dense), plain):
        assert a.keys() == b.keys()
        for k in a:
            ta, tb = (a[k].tensor, b[k].tensor) if hasattr(a[k], "tensor") else (a[k], b[k])
            assert torch.equal(ta, tb), k
    assert all(not r["instances"].has("pred_masks_rle") for r in dense)
    res = run("rle")
    assert len(getattr(m, "_graphs", {})) == graphs          # same graph key, no new capture
    torch.cuda.synchronize()
    for b, r in enumerate(res):
        inst = r["instances"]
        assert torch.equal(inst.pred_masks, plain[b]["pred_masks"])
        rles = inst.pred_masks_rle
        hw = list(inst.pred_masks.shape[1:])
        assert len(rles) == inst.pred_masks.shape[0] and all(x["size"] == hw for x in rles)
        if mapper:
            assert hw == [[120, 160], [300, 400]][b]
        if rles:
            assert torch.equal(rle.decode(rles), (inst.pred_masks != 0).to(torch.uint8))
            assert rles[0] == R.encode_masks(inst.pred_masks[:1].cpu().numpy())[0]
