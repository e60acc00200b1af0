"""TEST INFRASTRUCTURE — generates tests/golden/* by running the UNMODIFIED reference
(a reference checkout, via oracle/ref_shims.py) in the build container.  The reference cannot travel to
the GPU box, so its outputs are committed as small fixtures together with this script.

    python oracle/gen_golden.py manifest      # state-dict key/shape manifest from the reference constructors
    python oracle/gen_golden.py msda          # core op vectors (recipe of ops/test.py:24-63, seed 3) + larger cases
    python oracle/gen_golden.py modules       # per-module outputs (swin, projector, phi, pixel decoder, predictor)
    python oracle/gen_golden.py e2e           # eval_seg end to end (small Phi, 192^2 and 320x256) panoptic + referring
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")

from oracle import ref_shims  # noqa: E402


def gen_manifest():
    m = ref_shims.build_reference_psalm("panoptic", num_hidden_layers=2)
    sd = m.state_dict()
    man = {k: [list(v.shape), str(v.dtype).replace("torch.", "")] for k, v in sd.items()}
    with open(os.path.join(GOLD, "state_dict_manifest_phi2layers.json"), "w") as f:
        json.dump(man, f, indent=0, sort_keys=True)
    print("manifest:", len(man), "tensors")


def _msda_case(seed, N, M, D, Lq, L, P, shapes, dtype=torch.float32, loc_range=(0.0, 1.0)):
    from psalm.model.mask_decoder.Mask2Former_Simplify.modeling.pixel_decoder.ops.functions.ms_deform_attn_func import \
        ms_deform_attn_core_pytorch
    torch.manual_seed(seed)
    shapes_t = torch.as_tensor(shapes, dtype=torch.long)
    S = int(shapes_t.prod(1).sum())
    value = torch.rand(N, S, M, D) * 0.01
    loc = torch.rand(N, Lq, M, L, P, 2) * (loc_range[1] - loc_range[0]) + loc_range[0]
    aw = torch.rand(N, Lq, M, L, P) + 1e-5
    aw /= aw.sum(-1, keepdim=True).sum(-2, keepdim=True)
    out64 = ms_deform_attn_core_pytorch(value.double(), shapes_t, loc.double(), aw.double())
    out32 = ms_deform_attn_core_pytorch(value, shapes_t, loc, aw)
    return dict(value=value.numpy(), shapes=shapes_t.numpy(), loc=loc.numpy(), aw=aw.numpy(),
                out_f64=out64.numpy(), out_f32=out32.numpy())


def gen_msda():
    ref_shims.install()
    # (1) exactly the reference's own test vectors: ops/test.py:24-31 (N,M,D=1,2,2; Lq,L,P=2,2,2;
    #     shapes [(6,4),(3,2)], torch.manual_seed(3), CPU generator) — first draw = the "double" check
    c = _msda_case(3, 1, 2, 2, 2, 2, 2, [(6, 4), (3, 2)])
    np.savez_compressed(os.path.join(GOLD, "msda_ops_test.npz"), **c)
    # (2) the production head geometry at reduced size, locations spilling outside [0,1] (zero padding)
    c = _msda_case(11, 1, 8, 32, 128, 3, 4, [(4, 6), (8, 12), (16, 24)], loc_range=(-0.2, 1.2))
    np.savez_compressed(os.path.join(GOLD, "msda_m8d32.npz"), **c)
    # (3) ragged: 4 levels, odd sizes, D not a multiple of 4
    c = _msda_case(5, 1, 3, 6, 37, 4, 4, [(3, 5), (7, 2), (1, 9), (4, 4)], loc_range=(-0.1, 1.1))
    np.savez_compressed(os.path.join(GOLD, "msda_ragged.npz"), **c)
    print("msda golden written")


if __name__ == "__main__":
    os.makedirs(GOLD, exist_ok=True)
    what = sys.argv[1] if len(sys.argv) > 1 else "all"
    with torch.no_grad():
        if what in ("manifest", "all"):
            gen_manifest()
        if what in ("msda", "all"):
            gen_msda()
        if what in ("modules", "all"):
            from oracle import gen_golden_modules
            gen_golden_modules.main()
