"""Every producer of split planes writes, for every plane-set code, exactly the split of the fp32 value it writes
itself: the planes are compared bit for bit with a torch restatement of the split (csrc/common.cuh)."""
import ctypes as C

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]

if not torch.cuda.is_available():  # collected on CPU, skipped (never run without -m gpu anyway)
    pytest.skip("needs CUDA", allow_module_level=True)

from oobleck_b200 import lib as L  # noqa: E402
from oobleck_b200 import ops  # noqa: E402

DEV = "cuda"
CODES = [1, 2, 3, L.PLANES_BF16X3_FP16_PAIR, L.PLANES_FP16_PAIR]


def P(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def S():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def ref_planes(x: torch.Tensor, code: int) -> torch.Tensor:
    """16-bit patterns [planes_count(code), *x.shape] of the split of fp32 ``x``."""
    p0 = x.bfloat16()
    p1 = (x - p0.float()).bfloat16()
    p2 = (x - p0.float() - p1.float()).bfloat16()
    h0 = x.clamp(-65504, 65504).half()
    h1 = ((x - h0.float()) * 2048).clamp(-65504, 65504).half()
    bf16 = [p.view(torch.int16) for p in (p0, p1, p2)]
    pair = [h.view(torch.int16) for h in (h0, h1)]
    if code == L.PLANES_FP16_PAIR:
        return torch.stack(pair)
    if code == L.PLANES_BF16X3_FP16_PAIR:
        return torch.stack(bf16 + pair)
    return torch.stack(bf16[:code])


def new_planes(code: int, *shape) -> torch.Tensor:
    """A plane buffer filled with NaN patterns, so that a plane nobody writes cannot pass."""
    return torch.full((L.planes_count(code), *shape), float("nan"), dtype=torch.bfloat16, device=DEV)


def assert_split_of(planes: torch.Tensor, value: torch.Tensor, code: int, what: str) -> None:
    want = ref_planes(value, code)
    got = planes.view(torch.int16)
    for i in range(want.shape[0]):
        bad = int((got[i] != want[i]).sum())
        assert bad == 0, f"{what}, code {code}: plane {i} differs in {bad} of {want[i].numel()} elements"


def wide_randn(*shape):
    """Magnitudes from 1e-4 to 1e3: fp16-subnormal residuals, saturating pairs at the top of the range."""
    x = torch.randn(*shape, device=DEV)
    return x * torch.logspace(-4, 3, x.shape[-1], device=DEV) * 40


@pytest.mark.parametrize("code", CODES)
def test_split_planes(code):
    n = 1003
    x = wide_randn(n)
    ps = (n + 7) // 8 * 8
    planes = new_planes(code, ps)
    L.call("oob_split_planes", P(x), P(planes), n, ps, code, S())
    assert_split_of(planes[:, :n], x, code, "oob_split_planes")


@pytest.mark.parametrize("code", CODES)
def test_layernorm_fwd_bwd(code):
    rows, E = 37, 768
    x = torch.randn(rows, E, device=DEV) * 3 + 0.5
    g, b = torch.randn(E, device=DEV), torch.randn(E, device=DEV)
    y, mean, rstd = torch.empty_like(x), torch.empty(rows, device=DEV), torch.empty(rows, device=DEV)
    yp = new_planes(code, rows, E)
    L.call("oob_layernorm_fwd", P(x), P(g), P(b), P(y), P(yp), yp.stride(0), code, P(mean), P(rstd), rows, E, 1e-5,
           S())
    assert_split_of(yp, y, code, "layernorm forward")
    dy, dres = torch.randn(rows, E, device=DEV) * 1e3, torch.randn(rows, E, device=DEV)
    dx = torch.empty_like(x)
    dxp = new_planes(code, rows, E)
    dg, db = torch.zeros(E, device=DEV), torch.zeros(E, device=DEV)
    part = torch.empty(L.load().oob_ln_bwd_partials_floats(E), device=DEV)
    L.call("oob_layernorm_bwd", P(dy), P(x), P(mean), P(rstd), P(g), P(dres), P(dx), P(dxp), dxp.stride(0), code, P(dg),
           P(db), P(part), rows, E, 1.0, S())
    assert_split_of(dxp, dx, code, "layernorm backward")


@pytest.mark.parametrize("code", CODES)
@pytest.mark.parametrize("N", [256, 203])   # 256: 8-byte plane stores; 203: the per-element edge path
def test_gemm_epilogue(code, N):
    M, K = 192, 128
    A, W = torch.randn(M, K, device=DEV), torch.randn(N, K, device=DEV) * 0.05
    bias, R = torch.randn(N, device=DEV), wide_randn(M, N)
    d = torch.empty(M, N, device=DEV)
    planes = new_planes(code, M, N)
    ops.gemm(ops.split(A), False, ops.split(W), False, M, N, K, d=d, bias=bias, resid=R, planes_out=planes,
             planes_code=code)
    assert_split_of(planes, d, code, f"GEMM epilogue, N={N}")


@pytest.mark.parametrize("code", CODES)
def test_attention_fwd_bwd(code):
    B, T, H, D = 2, 100, 2, 64
    E = H * D
    torch.manual_seed(3)
    qkv = torch.randn(B * T, 3 * E, device=DEV)
    qp = ops.split(qkv)
    out, lse = torch.empty(B * T, E, device=DEV), torch.empty(B, H, T, device=DEV)
    outp = new_planes(code, B * T, E)
    L.call("oob_attention_fwd", P(qp), qp.stride(0), 0, P(out), P(outp), outp.stride(0), code, P(lse), B, T, H, D, S())
    assert_split_of(outp, out, code, "attention forward")
    dout = torch.randn(B * T, E, device=DEV) * 100
    dop = ops.split(dout)
    delta = torch.empty(B, H, T, device=DEV)
    dqkv = torch.empty(B * T, 3 * E, device=DEV)
    dqp = new_planes(code, B * T, 3 * E)
    L.call("oob_attention_bwd", P(qp), qp.stride(0), 0, P(out), P(dout), P(dop), dop.stride(0), P(lse), P(delta),
           P(dqkv), P(dqp), dqp.stride(0), code, B, T, H, D, S())
    assert_split_of(dqp, dqkv, code, "attention backward")


@pytest.mark.parametrize("code", CODES)
def test_adamw(code):
    n = 1003
    p, g = wide_randn(n), torch.randn(n, device=DEV)
    m, v = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    ps = (n + 7) // 8 * 8
    planes = new_planes(code, ps)
    L.call("oob_adamw_step", P(p), P(g), P(m), P(v), P(planes), ps, code, n, 1e-3, 0.9, 0.999, 1e-8, 0.01, 1, S())
    assert_split_of(planes[:, :n], p, code, "adamw")


def test_cross_entropy_plane_sets_agree():
    """The gradient has no fp32 copy to compare with: the plane sets of one call must nest instead."""
    B, T, V = 2, 17, 1000
    Vp = (V + 63) // 64 * 64
    torch.manual_seed(4)
    logits = torch.randn(B * T, Vp, device=DEV) * 3
    labels = torch.randint(0, V, (B, T), device=DEV)
    row_loss, loss = torch.empty(B * T, device=DEV), torch.zeros(1, device=DEV)
    got = {}
    for code in CODES:
        dp = new_planes(code, B * T, Vp)
        L.call("oob_cross_entropy", P(logits), Vp, P(labels), B, T, V, P(row_loss), P(loss), None, P(dp), Vp,
               dp.stride(0), code, 4096.0, S())
        got[code] = dp.view(torch.int16)
    bf16x3, pair = got[3], got[L.PLANES_FP16_PAIR]
    assert torch.equal(got[L.PLANES_BF16X3_FP16_PAIR], torch.cat([bf16x3, pair]))
    assert torch.equal(got[1], bf16x3[:1]) and torch.equal(got[2], bf16x3[:2])


def test_unknown_code_is_rejected():
    x = torch.randn(64, device=DEV)
    planes = torch.empty(4, 64, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(L.OobleckB200Error, match="plane-set code"):
        L.call("oob_split_planes", P(x), P(planes), 64, 64, 4, S())
