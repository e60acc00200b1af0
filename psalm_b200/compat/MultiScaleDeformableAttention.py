"""Drop-in for the reference's pybind extension module of the same name
(ops/setup.py:60, ops/src/vision.cpp:18-21).  Put this directory on PYTHONPATH and the reference's
`MSDeformAttnFunction.forward` (ops/functions/ms_deform_attn_func.py:34-39) runs on the sm_90a
kernel unmodified.  See INTEGRATION.md."""
from psalm_b200.msda import ms_deform_attn_backward, ms_deform_attn_forward  # noqa: F401
