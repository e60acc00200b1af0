"""Fused-epilogue linear layers on the Hopper tensor cores (wgmma, csrc/gemm_wgmma.cu) against a plain PyTorch fp32 evaluation of
the same op on the same 16-bit inputs: Swin `Mlp.fc1` + exact-erf GELU (swin_trans.py:37-44), MSDeformAttn `value_proj`
stored head-major (ms_deform_attn.py:95-99), plain bias.  Tolerance: the result is rounded once to 16 bits (rel 2^-9 bf16 /
2^-12 fp16) on top of fp32 accumulation; asserted as |err| <= rtol * |ref| + atol with atol tied to the output scale."""
import pytest
import torch

pytestmark = pytest.mark.gpu

TOL = {torch.bfloat16: 6e-3, torch.float16: 8e-4}
SHAPES = [  # (M, N, K)
    (1000, 256, 64),      # M tail inside one tile, single k-block
    (4096, 512, 128),     # Swin stage-0 fc1 shape (cut down in M)
    (777, 1024, 512),     # ragged M, 8 k-blocks (ring wraps twice)
    (40000, 256, 256),    # more tiles than SMs: persistent loop + both accumulators
    (300, 4096, 1024),    # stage-3 fc1
]


def _data(M, N, K, dt, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, K, generator=g).to(dt).cuda()
    w = (torch.randn(N, K, generator=g) * K ** -0.5).to(dt).cuda()
    b = torch.randn(N, generator=g).to(dt).cuda()
    return x, w, b


def _close(out, ref, dt):
    err = (out.float() - ref).abs()
    bound = TOL[dt] * ref.abs() + TOL[dt] * 0.05 * ref.abs().max()
    assert bool((err <= bound).all()), "max err %.3e at ref %.3e" % (float(err.max()), float(ref.flatten()[err.argmax()]))


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16], ids=["bf16", "f16"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "%dx%dx%d" % s)
@pytest.mark.parametrize("epi", ["bias", "gelu_erf"])
def test_linear_fused_vs_fp32(shape, dt, epi):
    from psalm_b200 import kernels
    M, N, K = shape
    x, w, b = _data(M, N, K, dt, 1)
    assert kernels.linear_fused_supported(x, w, epi)
    out = kernels.linear_fused(x, w, b, epi)
    ref = x.float() @ w.float().t() + b.float()
    if epi == "gelu_erf":
        ref = torch.nn.functional.gelu(ref)
    assert out.shape == (M, N) and out.dtype == dt
    _close(out, ref, dt)


def test_gelu_epilogue_over_the_whole_input_range():
    """K = 64 with one-hot rows: the accumulator IS a chosen value, so the epilogue's erfc polynomial is swept over
    [-12, 12] including the clamp region; asserted against float64 erf after the 16-bit rounding of the output."""
    from psalm_b200 import kernels
    dt = torch.float16
    M, N, K = 4096, 256, 64
    vals = torch.linspace(-12, 12, M)
    x = torch.zeros(M, K)
    x[:, 0] = vals
    w = torch.zeros(N, K)
    w[:, 0] = torch.linspace(0.25, 1.0, N)
    x, w = x.to(dt).cuda(), w.to(dt).cuda()
    out = kernels.linear_fused(x, w, None, "gelu_erf")
    pre = x.double()[:, :1] * w.double()[:, 0][None]
    ref = 0.5 * pre * (1 + torch.erf(pre / 2 ** 0.5))
    err = (out.double() - ref).abs()
    assert bool((err <= 6e-4 * ref.abs() + 1e-6).all()), float(err.max())


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16], ids=["bf16", "f16"])
def test_head_major_epilogue_is_the_value_layout(dt):
    from psalm_b200 import kernels
    B, S, C = 3, 1376, 256             # S % 32 == 0 (a warp's 32 rows stay inside one image), S % 128 != 0
    x, w, b = _data(B * S, C, C, dt, 2)
    assert kernels.linear_fused_supported(x, w, "head_major", S) and not kernels.linear_fused_supported(x, w, "head_major", 1350)
    x = x.view(B, S, C)
    out = kernels.linear_fused(x, w, b, "head_major", S)
    assert out.shape == (B, 8, S, 32)
    ref = (x.float() @ w.float().t() + b.float()).view(B, S, 8, 32).permute(0, 2, 1, 3)
    _close(out, ref, dt)


def test_row_strided_input_view_and_unsupported_shapes():
    from psalm_b200 import _lib, kernels
    dt = torch.bfloat16
    x, w, b = _data(512, 256, 128, dt, 3)
    wide = torch.randn(512, 384).to(dt).cuda()
    wide[:, 128:256] = x
    out = kernels.linear_fused(wide[:, 128:256], w, b, "bias")      # row stride 384, no copy
    _close(out, x.float() @ w.float().t() + b.float(), dt)
    assert not kernels.linear_fused_supported(x, w[:200], "bias")    # N % 256
    assert not kernels.linear_fused_supported(x.float(), w.float(), "bias")
    with pytest.raises(_lib.PsalmKernelError):
        kernels.linear_fused(x, w[:200].contiguous(), b[:200].contiguous(), "bias")
