"""TEST INFRASTRUCTURE — import shims that let the *unmodified* reference (a reference checkout named by PSALM_REFERENCE_ROOT,
zamling/PSALM) run on CPU in the build container.  Used only by `oracle/gen_golden.py` (fixture
generation) and by `tests/test_oracle_vs_reference.py` (skipped when the reference is absent, e.g.
on the GPU box).  Nothing in `psalm_b200/` imports this file.

The reference imports detectron2 / timm / fvcore / addict / pycocotools / panopticapi /
MultiScaleDeformableAttention at module-import time (llava_phi.py:2,18-32); none are installed.
We fabricate the few symbols the inference path *executes* (SURVEY.md §8c) and auto-mock the rest.
The MultiScaleDeformableAttention stub raises, so the reference falls through its own bare
`except:` (ops/modules/ms_deform_attn.py:117-119) to `ms_deform_attn_core_pytorch` — the
reference's real CPU path.
"""
import importlib.abc
import importlib.machinery
import os
import sys
import types

import torch
import torch.nn.functional as F

REFERENCE_ROOT = os.environ.get("PSALM_REFERENCE_ROOT", "")

_FAKE_ROOTS = ("detectron2", "pycocotools", "panopticapi", "timm", "fvcore", "addict",
               "MultiScaleDeformableAttention", "shortuuid", "iopath", "matplotlib")


_SUBMODULES = ("transforms", "detection_utils", "mask", "comm", "data", "utils", "structures",
               "modeling", "config", "projects", "point_rend", "evaluation", "layers", "models", "nn")


def reference_available():
    return bool(REFERENCE_ROOT) and os.path.isdir(os.path.join(REFERENCE_ROOT, "psalm"))


class _AutoMock(types.ModuleType):
    """Module whose every missing attribute is a callable, subscriptable dummy class."""

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        if name in _SUBMODULES:
            import importlib
            sub = importlib.import_module(self.__name__ + "." + name)
            setattr(self, name, sub)
            return sub
        dummy = type(name, (), {"__init__": lambda self, *a, **k: None,
                                "__call__": lambda self, *a, **k: None})
        setattr(self, name, dummy)
        return dummy


class _Finder(importlib.abc.MetaPathFinder, importlib.abc.Loader):
    def find_spec(self, fullname, path=None, target=None):
        if fullname.split(".")[0] in _FAKE_ROOTS and fullname not in sys.modules:
            return importlib.machinery.ModuleSpec(fullname, self, is_package=True)
        return None

    def create_module(self, spec):
        m = _AutoMock(spec.name)
        m.__path__ = []
        return m

    def exec_module(self, module):
        _populate(module)


class _AttrDict(dict):
    """addict.Dict stand-in (recursive attribute dict)."""

    def __init__(self, *args, **kwargs):
        super().__init__()
        for k, v in dict(*args, **kwargs).items():
            self[k] = self._conv(v)

    @classmethod
    def _conv(cls, v):
        if isinstance(v, dict) and not isinstance(v, cls):
            return cls(v)
        if isinstance(v, (list, tuple)):
            return type(v)(cls._conv(x) for x in v)
        return v

    def __setitem__(self, k, v):
        super().__setitem__(k, self._conv(v))

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            return self.__missing__(k)

    def __missing__(self, k):
        v = type(self)()
        super().__setitem__(k, v)
        return v

    def __setattr__(self, k, v):
        self[k] = v


class Instances:
    """detectron2.structures.Instances stand-in: attribute bag with image_size."""

    def __init__(self, image_size, **kw):
        object.__setattr__(self, "_image_size", image_size)
        object.__setattr__(self, "_fields", {})
        for k, v in kw.items():
            self._fields[k] = v

    @property
    def image_size(self):
        return self._image_size

    def __setattr__(self, k, v):
        self._fields[k] = v

    def __getattr__(self, k):
        f = object.__getattribute__(self, "_fields")
        if k in f:
            return f[k]
        raise AttributeError(k)

    def get_fields(self):
        return self._fields


class Boxes:
    def __init__(self, tensor):
        self.tensor = tensor


class BitMasks:
    def __init__(self, tensor):
        self.tensor = tensor


class ImageList:
    """detectron2.structures.ImageList.from_tensors restated (detectron2 v0.6 semantics: pad each
    image at bottom/right to the max size rounded up to `size_divisibility`)."""

    def __init__(self, tensor, image_sizes):
        self.tensor = tensor
        self.image_sizes = image_sizes

    @staticmethod
    def from_tensors(tensors, size_divisibility=0, pad_value=0.0):
        sizes = [tuple(t.shape[-2:]) for t in tensors]
        mh = max(s[0] for s in sizes)
        mw = max(s[1] for s in sizes)
        if size_divisibility > 1:
            d = size_divisibility
            mh = (mh + d - 1) // d * d
            mw = (mw + d - 1) // d * d
        out = tensors[0].new_full((len(tensors),) + tuple(tensors[0].shape[:-2]) + (mh, mw), pad_value)
        for i, t in enumerate(tensors):
            out[i, ..., : t.shape[-2], : t.shape[-1]].copy_(t)
        return ImageList(out, sizes)


def sem_seg_postprocess(result, img_size, output_height, output_width):
    """detectron2.modeling.postprocessing.sem_seg_postprocess restated (v0.6)."""
    result = result[:, : img_size[0], : img_size[1]].expand(1, -1, -1, -1)
    return F.interpolate(result, size=(output_height, output_width), mode="bilinear", align_corners=False)[0]


def _populate(m):
    n = m.__name__
    if n == "timm.models.layers":
        m.DropPath = lambda p=0.0: torch.nn.Identity()
        m.to_2tuple = lambda x: x if isinstance(x, (tuple, list)) else (x, x)
        m.trunc_normal_ = lambda t, std=1.0, **k: torch.nn.init.trunc_normal_(t, std=std, a=-2 * std, b=2 * std)
    elif n == "fvcore.nn.weight_init" or n == "fvcore.nn":
        def c2_xavier_fill(mod):
            torch.nn.init.kaiming_uniform_(mod.weight, a=1)
            if mod.bias is not None:
                torch.nn.init.constant_(mod.bias, 0)
        target = m
        if n == "fvcore.nn":
            return
        target.c2_xavier_fill = c2_xavier_fill
        target.c2_msra_fill = c2_xavier_fill
    elif n == "addict":
        m.Dict = _AttrDict
    elif n == "detectron2.structures":
        m.Instances, m.Boxes, m.BitMasks, m.ImageList = Instances, Boxes, BitMasks, ImageList
        m.BoxMode = type("BoxMode", (), {"XYXY_ABS": 0, "XYWH_ABS": 1})
        m.PolygonMasks = type("PolygonMasks", (), {})
    elif n == "detectron2.modeling.postprocessing":
        m.sem_seg_postprocess = sem_seg_postprocess
    elif n == "detectron2.utils.memory":
        m.retry_if_cuda_oom = lambda f: f
    elif n == "detectron2.config":
        m.configurable = lambda f=None, **k: (f if f is not None else (lambda g: g))
    elif n == "MultiScaleDeformableAttention":
        def _raise(*a, **k):
            raise RuntimeError("reference CUDA op not built (oracle shim): falling back to core_pytorch")
        m.ms_deform_attn_forward = _raise
        m.ms_deform_attn_backward = _raise


_installed = False


def install():
    """Idempotently install the import shims and put the reference on sys.path."""
    global _installed
    if _installed:
        return
    if not reference_available():
        raise RuntimeError("reference tree not present at %s" % REFERENCE_ROOT)
    sys.meta_path.insert(0, _Finder())
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    _installed = True


def _merge(a, b):
    for k, v in b.items():
        if isinstance(v, dict) and isinstance(a.get(k), dict):
            _merge(a[k], v)
        else:
            a[k] = v
    return a


def load_mask_cfg(seg_task="panoptic", name="maskformer2_swin_base_384_bs16_50ep.yaml"):
    """YAML `_BASE_` merge of psalm/mask_config (train_datasets.py:36-42 uses fvcore CfgNode)."""
    import yaml
    d = os.path.join(REFERENCE_ROOT, "psalm", "mask_config")

    def load(fn):
        with open(os.path.join(d, fn)) as f:
            cur = yaml.unsafe_load(f)
        base = cur.pop("_BASE_", None)
        if base:
            return _merge(load(os.path.basename(base)), cur)
        return cur

    cfg = _AttrDict(load(name))
    cfg.MODEL.MASK_FORMER.SEG_TASK = seg_task
    return cfg


def build_reference_psalm(seg_task="panoptic", num_hidden_layers=None, hidden_size=None, davis=False, **cfg_over):
    """Construct the reference `PSALM` (llava_phi.py:146; `davis`: PSALMForDAVISEval, :1477) on CPU, fp32, eval mode."""
    install()
    from psalm.model.language_model.llava_phi import LlavaConfig
    if davis:
        from psalm.model.language_model.llava_phi import PSALMForDAVISEval as PSALM
    else:
        from psalm.model.language_model.llava_phi import PSALM
    kw = {}
    if num_hidden_layers is not None:
        kw["num_hidden_layers"] = num_hidden_layers
    if hidden_size is not None:
        kw.update(hidden_size=hidden_size, intermediate_size=4 * hidden_size,
                  num_attention_heads=hidden_size // 64)
    kw.update(cfg_over)
    config = LlavaConfig(**kw)
    config.mm_vision_tower = "swin"
    config.swin_type = "base"
    config.mm_projector_type = "swin_conv"
    config.projector_outdim = config.hidden_size
    config.mm_input_embeds = 1024
    config.mask_decode_train = True
    config._attn_implementation = "eager"
    cfg = load_mask_cfg(seg_task)
    model = PSALM(config, mask_decoder_cfg=cfg)
    model.train(False)
    model.float()
    return model
