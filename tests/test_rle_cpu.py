"""COCO RLE without a GPU: the numpy restatement of pycocotools (oracle/coco_rle.py) on hand-checkable vectors, round
trips, the ragged multi-rank gather, and the mask_format plumbing of eval_seg with the device encoder replaced by the
oracle."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import coco_rle as R
from psalm_b200 import dist as PD
from psalm_b200 import rle
from psalm_b200 import psalm as P
from psalm_b200.structures import Boxes, Instances

HAND = [
    (np.zeros((2, 2)), [4], b"4"),
    (np.ones((2, 2)), [0, 4], b"04"),
    (np.array([[1, 0], [0, 0]]), [0, 1, 3], b"013"),
    (np.array([[0, 1, 0], [1, 1, 1], [1, 1, 1]]), [1, 5, 1, 2], b"151M"),   # negative delta cnt[3] - cnt[1]
    (np.zeros((4, 4)), [16], b"`0"),                                       # 16 has bit 0x10 set: a second group
]


@pytest.mark.parametrize("mask,counts,string", HAND)
def test_hand_vectors(mask, counts, string):
    assert R.encode(mask) == counts
    assert R.to_string(counts) == string
    assert R.fr_string(string) == counts
    assert R.fr_string(string.decode()) == counts
    assert np.array_equal(R.decode(counts, *mask.shape), (mask != 0).astype(np.uint8))


def test_large_empty_mask():
    assert R.to_string(R.encode(np.zeros((1024, 1024), np.uint8))) == b"PPPP1"


def _random_masks(rng):
    out = []
    for H, W in ((1, 1), (1, 9), (9, 1), (7, 33), (31, 17)):
        for p in (0.0, 0.01, 0.5, 0.99, 1.0):
            out.append((rng.random((H, W)) < p).astype(np.uint8))
    y, x = np.mgrid[:6, :5]
    out.append(((x * 6 + y) % 2).astype(np.uint8))   # Fortran-order checkerboard: every run has length 1
    return out


def test_oracle_round_trip_area_bbox():
    rng = np.random.default_rng(0)
    for m in _random_masks(rng):
        H, W = m.shape
        c = R.encode(m)
        assert sum(c) == H * W and all(v > 0 for v in c[1:])
        assert R.fr_string(R.to_string(c)) == c
        assert np.array_equal(R.decode(c, H, W), m)
        assert R.area(c) == int(m.sum())
        ys, xs = np.nonzero(m)
        want = [0.0] * 4 if m.sum() == 0 else [xs.min(), ys.min(), xs.max() - xs.min() + 1, ys.max() - ys.min() + 1]
        assert R.to_bbox(c, H, W) == [float(v) for v in want]


def test_against_pycocotools_when_installed():
    mask_util = pytest.importorskip("pycocotools.mask")
    rng = np.random.default_rng(1)
    masks = [m for m, _, _ in HAND] + _random_masks(rng)
    for m in masks:
        m = m.astype(np.uint8)
        ref = mask_util.encode(np.asfortranarray(m[:, :, None]))[0]
        assert R.to_string(R.encode(m)) == ref["counts"]
        assert R.area(R.encode(m)) == int(mask_util.area(ref))
        assert R.to_bbox(R.encode(m), *m.shape) == [float(v) for v in mask_util.toBbox(ref)]


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _payload(rank):
    if rank == 1:   # an empty rank: no masks at all
        return torch.empty(0, dtype=torch.uint8), torch.zeros(1, dtype=torch.int64)
    strs = [b"04", b"151M", b"PPPP1"]
    chars = torch.tensor(list(b"".join(strs)), dtype=torch.uint8)
    return chars, torch.tensor([0, 2, 6, 11], dtype=torch.int64)


def _worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    if rank == 2:
        chars, offs = torch.tensor(list(b"013"), dtype=torch.uint8), torch.tensor([0, 3], dtype=torch.int64)
    else:
        chars, offs = _payload(rank)
    got = PD.gather_rle(chars, offs)
    q.put((rank, [(bytes(c.tolist()), o.tolist()) for c, o in got]))
    dist.destroy_process_group()


def test_gather_rle_three_ranks_ragged_and_empty():
    world = 3
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in range(world))
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    want = [(b"04151MPPPP1", [0, 2, 6, 11]), (b"", [0]), (b"013", [0, 3])]
    for _, got in res:
        assert got == want


def test_gather_rle_without_process_group_is_identity():
    c, o = _payload(0)
    [(c2, o2)] = PD.gather_rle(c, o)
    assert c2 is c and o2 is o


def _oracle_encode_device(masks):
    parts = [masks] if isinstance(masks, torch.Tensor) else list(masks)
    H, W = parts[0].shape[-2:]
    strs = [R.to_string(R.encode(m.numpy())) for t in parts for m in t.reshape(-1, H, W)]
    offs = np.concatenate(([0], np.cumsum([len(s) for s in strs]))).astype(np.int64)
    return dict(size=(int(H), int(W)), chars=torch.tensor(list(b"".join(strs)), dtype=torch.uint8),
                offsets=torch.from_numpy(offs))


class _Stream:
    def wait_event(self, e):
        pass


class _Done:
    def synchronize(self):
        pass


class _Model:
    device = "cpu"

    def __init__(self, results):
        self.results = results

    def post_process(self, out, image_hw, seg_info, boxes=None, hostvecs=None, is_thing_list=None,
                     object_mask_threshold=None, overlap_threshold=None):
        return self.results


def _results():
    g = torch.Generator().manual_seed(0)
    out = []
    for H, W in ((6, 5), (6, 5), (4, 7)):   # two images of one size, one of another (the mapper flow)
        inst = Instances((H, W))
        inst.pred_masks = (torch.rand(3, H, W, generator=g) > 0.5).float()
        inst.pred_boxes = Boxes(torch.zeros(3, 4))
        inst.scores = torch.tensor([0.9, 0.5, 0.25])
        inst.pred_classes = torch.tensor([1, 2, 3])
        out.append({"instances": inst, "sem_seg": torch.zeros(2, H, W)})
    out.append({"sem_seg": torch.zeros(2, 3, 3)})   # a result without instances is left alone
    return out


def _pending(results, mask_format):
    return P.PendingSeg(_Model(results), [(None, None, None)], (6, 5), None, None, _Done(), (0.8, 0.8), mask_format)


def test_pending_seg_mask_format_dense_and_rle(monkeypatch):
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: _Stream())
    calls = []
    monkeypatch.setattr(rle, "encode_device", lambda m: calls.append(len(m)) or _oracle_encode_device(m))
    res = _results()
    snapshot = [{k: v for k, v in r.items()} for r in res]
    got = _pending(res, "dense").result()
    assert got is res and calls == []
    assert all(not r["instances"].has("pred_masks_rle") for r in got if "instances" in r)
    assert all(r.keys() == s.keys() and all(r[k] is s[k] for k in r) for r, s in zip(got, snapshot))

    got = _pending(_results(), "rle").result()
    assert sorted(calls) == [1, 2]   # one batch per output size
    for r in got:
        if "instances" not in r:
            continue
        inst = r["instances"]
        want = R.encode_masks(inst.pred_masks.numpy())
        assert inst.pred_masks_rle == want and inst.pred_masks.dtype == torch.float32
        recs = rle.instances_to_coco_json(inst, 7)
        assert [x["segmentation"]["counts"] for x in recs] == [w["counts"].decode() for w in want]
        assert recs[0]["bbox"] == [0.0, 0.0, 0.0, 0.0] and recs[1]["category_id"] == 2 and recs[2]["score"] == 0.25
        assert all(x["image_id"] == 7 and x["segmentation"]["size"] == list(inst.image_size) for x in recs)


def test_mask_format_is_checked_and_defaults_to_dense():
    import inspect
    for fn in (P.PSALM.eval_seg, P.PSALM.eval_seg_async):
        assert inspect.signature(fn).parameters["mask_format"].default == "dense"
    with pytest.raises(ValueError, match="mask_format"):
        P.PSALM.eval_seg_async(object(), images=None, mask_format="png")


def test_cpu_masks_are_rejected():
    from psalm_b200 import _lib
    with pytest.raises(_lib.PsalmKernelError):
        rle.encode(torch.zeros(2, 4, 4))


def test_instances_to_coco_json_boxes_come_from_pred_boxes():
    inst = Instances((4, 4))
    inst.pred_masks = torch.zeros(1, 4, 4)
    inst.pred_boxes = Boxes(torch.tensor([[1.0, 2.0, 4.0, 3.5]]))
    inst.scores = torch.tensor([0.5])
    inst.pred_classes = torch.tensor([3])
    inst.pred_masks_rle = [{"size": [4, 4], "counts": b"`0"}]
    [rec] = rle.instances_to_coco_json(inst, 1)
    assert rec == {"image_id": 1, "category_id": 3, "bbox": [1.0, 2.0, 3.0, 1.5], "score": 0.5,
                   "segmentation": {"size": [4, 4], "counts": "`0"}}
    assert rle.instances_to_coco_json(Instances((4, 4)), 1) == []
