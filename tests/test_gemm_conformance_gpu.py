"""Conformance of the split-plane GEMM (csrc/gemm_sm90.cuh, csrc/gemm.cu) at the edges the model reaches.

Every operand is read through a padded view: a plane buffer larger than the logical matrix, at an offset, with a
plane stride larger than rows * ld, whose every slot outside the matrix holds a NaN pattern.  A kernel that reads past
the GEMM's extents therefore produces NaN.  Every output is written into a guarded buffer whose slots outside [M, N]
hold a sentinel that must survive.  Values are checked per element against fp64:

    |d - A@B| <= bound * (|A| @ |B|) + floor

|A| @ |B| is the error scale of a dot product; for same-sign data it equals |A@B|, where the chunked round-to-nearest
promotion of the main accumulator matters most.  Each bound sits about 4x above the worst ratio measured on one
NVIDIA H100 80GB HBM3 (700 W power limit); the measured figure is given next to it.
"""
import ctypes as C

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

if not torch.cuda.is_available():  # collected on CPU, skipped (never run without -m gpu anyway)
    pytest.skip("needs CUDA", allow_module_level=True)

from oobleck_b200 import lib as L  # noqa: E402
from oobleck_b200 import ops  # noqa: E402
from oracle import gpt2 as og  # noqa: E402

DEV = "cuda"
NAN16 = 0x7FC0          # NaN as bf16 and as fp16: the padding of every operand view
SENTINEL = 0x7FC0DEAD   # NaN with a payload: the guard band of every fp32 output
PAIR_FLOOR = 2.0 ** -36  # absolute error of one fp16-pair element below the fp16 normal range (test_split5_fp16_pair)

# Operand formats: (plane-set code of the buffer, nsplit, fp16 pair at planes 3-4, fp16 pair at planes 0-1)
FMT = {
    "bf16x1": (L.PLANES_BF16X3_FP16_PAIR, 1, False, False),
    "bf16x2": (L.PLANES_BF16X3_FP16_PAIR, 2, False, False),
    "bf16x3": (L.PLANES_BF16X3_FP16_PAIR, 3, False, False),
    "pair3x1": (L.PLANES_BF16X3_FP16_PAIR, 1, True, False),
    "pair3x2": (L.PLANES_BF16X3_FP16_PAIR, 2, True, False),
    "pair0x2": (L.PLANES_FP16_PAIR, 2, False, True),
}
# What stage.cu's formats() reads: bf16 x 3 (3-plane buffers) or the pair-only buffers of an fp16 backward.
STAGE_FMT = {"bf16x3": (3, 3, False, False), "pair0x2": (L.PLANES_FP16_PAIR, 2, False, True)}

# Per-element bounds on |d - A@B| / (|A| @ |B|).  Comment: the worst ratio measured over every GEMM that uses the
# bound (tile sweep, LM head, weight views, wide range, many waves, cache eviction).  The two fp16-pair layouts read the
# same values and share a bound.
BOUND = {
    "bf16x1": 8e-3,     # 2.0e-3 (tile sweep)
    "bf16x2": 3e-5,     # 8.2e-6 (tile sweep)
    "bf16x3": 1e-6,     # 2.4e-7 (LM-head wgrad; tile sweep 2.3e-7)
    "pair3x1": 2e-3,    # 4.3e-4 (tile sweep)
    "pair3x2": 1.5e-6,  # 2.8e-7 (tile sweep)
    "pair0x2": 1.5e-6,  # 3.5e-7 (LM-head wgrad; tile sweep 2.8e-7)
}


def P(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def S():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def round8(n):
    return (n + 7) // 8 * 8


# ---- helpers -------------------------------------------------------------------------------------------------------

def operand(x, mn_major, code, pad_cols=8, pad_rows=8, offset=64, plane_gap=64):
    """The split of ``x`` (logical [mn, k]: A as [M, K], B as [N, K]) in a NaN-padded plane buffer.

    The matrix is stored [mn][k] (K-major) or [k][mn] (``mn_major``).  The returned view is
    [planes_count(code), rows + pad_rows, ld] with ld = round8(cols + pad_cols), starting ``offset`` elements into
    the buffer, with plane stride (rows + pad_rows) * ld + ``plane_gap``.  Hand it to ``ops.gemm``: its ``cols`` and
    ``ld`` are the padded width.  Every slot outside the matrix holds NAN16, written as raw bits."""
    assert offset % 8 == 0 and plane_gap % 8 == 0
    stored = (x.t() if mn_major else x).contiguous().float()
    rows, cols = stored.shape
    ld = round8(cols + pad_cols)
    prows = rows + pad_rows
    ps = prows * ld + plane_gap
    n = L.planes_count(code)
    flat = torch.full((offset + n * ps,), NAN16, dtype=torch.int16, device=DEV)
    view = flat.as_strided((n, prows, ld), (ps, ld, 1), offset)
    src = torch.zeros(rows, round8(cols), device=DEV)
    src[:, :cols] = stored
    view[:, :rows, :cols] = ops.split(src, nplanes=code).view(torch.int16)[:, :, :cols]
    return flat.view(torch.bfloat16).as_strided((n, prows, ld), (ps, ld, 1), offset)


def gemm(a, a_mn, b, b_mn, M, N, K, fmt, **kw):
    _, ns, fp16, pair0 = fmt
    ops.gemm(a, a_mn, b, b_mn, M, N, K, nsplit=ns, a_fp16=fp16, b_fp16=fp16, a_pair0=pair0, b_pair0=pair0, **kw)


def guarded(M, N, ldd=None, inner=None):
    """fp32 output [M + 8, ldd] (ldd >= N + 8) filled with SENTINEL; ``inner`` initialises [:M, :N]."""
    ldd = N + 8 if ldd is None else ldd
    assert ldd >= N + 8
    d = torch.empty(M + 8, ldd, device=DEV)
    d.view(torch.int32).fill_(SENTINEL)
    if inner is not None:
        d[:M, :N] = inner
    return d


def guarded_planes(code, M, N, ldp=None):
    ldp = round8(N) + 8 if ldp is None else ldp
    return torch.full((L.planes_count(code), M + 8, ldp), NAN16, dtype=torch.int16, device=DEV).view(torch.bfloat16)


def assert_guard(out, M, N, what=""):
    """Every element of ``out`` ([M + 8, ld] fp32 or [planes, M + 8, ld] 16-bit) outside [:M, :N] is untouched."""
    if out.dtype == torch.float32:
        bits, want = out.view(torch.int32), SENTINEL
    else:
        bits, want = out.view(torch.int16), NAN16
    outside = torch.ones_like(bits, dtype=torch.bool)
    outside[..., :M, :N] = False
    bad = int((bits[outside] != want).sum())
    assert bad == 0, f"{what}: {bad} elements written outside [{M}, {N}]"


def check_value(d, ref, scale, bound, floor=0.0, what=""):
    """Per element |d - ref| <= bound * scale + floor (fp64).  Returns the worst ratio (|d - ref| - floor) / scale,
    i.e. the smallest bound that would pass."""
    err = (d.double() - ref).abs()
    excess = (err - floor).clamp_min(0)
    ratio = torch.where(scale > 0, excess / scale.clamp_min(1e-300),
                        torch.where(excess > 0, torch.inf, 0.0).double())
    ratio = torch.nan_to_num(ratio, nan=torch.inf)
    worst = int(ratio.argmax())
    r = ratio.flatten()[worst].item()
    print(f"ratio {what} {r:.3e}")
    if r > bound:
        idx = [int(i) for i in torch.unravel_index(torch.tensor(worst), ratio.shape)]
        pytest.fail(f"{what}: worst element {idx}: got {d.flatten()[worst].item()!r}, want "
                    f"{ref.flatten()[worst].item()!r}, scale {scale.flatten()[worst].item():.3e}: ratio {r:.3e} > "
                    f"bound {bound:.1e}")
    return r


def check(d, A, B, bound, floor=0.0, what=""):
    """|d - A@B| <= bound * (|A| @ |B|) + floor per element, computed in fp64 on the GPU."""
    A64, B64 = A.double(), B.double()
    return check_value(d, A64 @ B64, A64.abs() @ B64.abs(), bound, floor, what)


def pair_floor(A, B):
    """The absolute fp16-pair error floor PAIR_FLOOR of every operand element, propagated through A @ B."""
    return PAIR_FLOOR * (A.double().abs().sum(1, keepdim=True) + B.double().abs().sum(0, keepdim=True))


# ---- 1. tiles, K tails and the pipeline ring -------------------------------------------------------------------------
# The ring holds 2 k-blocks for nsplit 3, 3 for nsplit 2 and 7 for nsplit 1 (227 KB of shared memory); the main
# accumulator is promoted every 8 k-blocks (GEMM_CHUNK_ELEMS = 512).  The set below covers each of 1, 2, 3, 7, 8 and 9
# k-blocks (below, at and above every ring depth, and across the first promotion chunk), the K tails 8, 24, 72 and
# 520, and odd K; M and N each take 1, 8, 127, 129 and 136 somewhere (one row or column, the smallest aligned size, one
# tile minus / plus one, a tile plus an 8-wide tail), each paired with a different K so that 12 shapes cover all of it.
# Every shape runs for all four major combinations and all six operand formats.
SWEEP = [
    (129, 136, 64), (127, 129, 128), (136, 127, 192), (1, 136, 448), (129, 8, 512), (8, 129, 576),
    (136, 1, 8), (127, 136, 24), (129, 127, 72), (136, 129, 520), (129, 136, 17), (127, 8, 1017),
]


@pytest.mark.parametrize("a_mn", [False, True])
@pytest.mark.parametrize("b_mn", [False, True])
@pytest.mark.parametrize("shape", SWEEP, ids=lambda s: "x".join(map(str, s)))
def test_tile_sweep(a_mn, b_mn, shape):
    M, N, K = shape
    torch.manual_seed(M * 7 + N * 3 + K)
    A, B = torch.randn(M, K, device=DEV), torch.randn(K, N, device=DEV)
    ops5 = (operand(A, a_mn, L.PLANES_BF16X3_FP16_PAIR), operand(B.t(), b_mn, L.PLANES_BF16X3_FP16_PAIR))
    ops22 = (operand(A, a_mn, L.PLANES_FP16_PAIR, offset=8), operand(B.t(), b_mn, L.PLANES_FP16_PAIR, plane_gap=8))
    for name, fmt in FMT.items():
        a, b = ops22 if fmt[0] == L.PLANES_FP16_PAIR else ops5
        d = guarded(M, N)
        gemm(a, a_mn, b, b_mn, M, N, K, fmt, d=d)
        assert_guard(d, M, N, name)
        floor = pair_floor(A, B) if "pair" in name else 0.0
        check(d[:M, :N], A, B, BOUND[name], floor, f"sweep {name}")


# ---- 2. LM-head shapes ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", list(STAGE_FMT))
def test_lm_head_shapes(fmt):
    """oob_head_forward / oob_head_backward at GPT-2 sizes: the contraction over V = 50257 reads a gradient buffer of
    row stride Vp = 50304 whose padding columns are NaN here (cross-entropy writes zeros there)."""
    V, Vp, E, T = 50257, 50304, 1600, 256
    f = STAGE_FMT[fmt]
    code = f[0]
    torch.manual_seed(11)
    lnf = torch.randn(T, E, device=DEV)
    W = torch.randn(V, E, device=DEV) * 0.02
    dlog = torch.randn(T, V, device=DEV) * 0.02
    lnf_op = operand(lnf, False, code, pad_cols=0, pad_rows=0, offset=0, plane_gap=0)
    # lm_head.weight [V, E] inside the flat parameter planes: offset 2E (ln_f), plane stride 2E + V E
    w_op = operand(W, False, code, pad_cols=0, pad_rows=0, offset=2 * E, plane_gap=2 * E)
    dlog_op = operand(dlog, False, code, pad_cols=Vp - V, pad_rows=0, offset=0, plane_gap=0)
    assert dlog_op.shape[2] == Vp
    bound = BOUND[fmt]
    pair = fmt.startswith("pair")
    # forward: logits [T, V] (ld Vp) = lnf . W^T
    d = guarded(T, V, ldd=Vp)
    gemm(lnf_op, False, w_op, False, T, V, E, f, d=d)
    assert_guard(d, T, V, "forward")
    check(d[:T, :V], lnf, W.t(), bound, pair_floor(lnf, W.t()) if pair else 0.0, f"lm_head forward {fmt}")
    del d
    # dgrad: dln [T, E] = dlog[:, :V] . W, W read N-major
    d = guarded(T, E)
    gemm(dlog_op, False, w_op, True, T, E, V, f, d=d)
    assert_guard(d, T, E, "dgrad")
    check(d[:T, :E], dlog, W, bound, pair_floor(dlog, W) if pair else 0.0, f"lm_head dgrad {fmt}")
    del d
    # wgrad: dW [V, E] += alpha . dlog^T . lnf, dlog read M-major
    alpha = 1.0 / 1024
    acc0 = torch.randn(V, E, device=DEV) * 1e-4
    d = guarded(V, E, inner=acc0)
    gemm(dlog_op, True, lnf_op, True, V, E, T, f, d=d, accumulate=True, alpha=alpha)
    assert_guard(d, V, E, "wgrad")
    A64, B64 = dlog.t().double(), lnf.double()
    ref = acc0.double() + alpha * (A64 @ B64)
    scale = acc0.double().abs() + alpha * (A64.abs() @ B64.abs())
    floor = alpha * pair_floor(dlog.t(), lnf) if pair else 0.0
    check_value(d[:V, :E], ref, scale, bound, floor, f"lm_head wgrad {fmt}")


# ---- 3. weight-style views -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", ["bf16x3", "pair3x2", "pair0x2"])
def test_weight_views(fmt):
    """A weight [K, N] as PlaneView::weight reads it: at an offset inside the flat parameter planes (ld = N), with the
    plane stride of the whole buffer.  Forward reads it N-major, dgrad K-major."""
    M, K, N = 200, 320, 456
    f = FMT[fmt]
    torch.manual_seed(13)
    X, W, dY = torch.randn(M, K, device=DEV), torch.randn(K, N, device=DEV) * 0.05, torch.randn(M, N, device=DEV)
    w_op = operand(W.t(), True, f[0], pad_cols=0, pad_rows=0, offset=8 * 1001, plane_gap=8 * 4321)
    pair = fmt.startswith("pair")
    d = guarded(M, N)
    gemm(operand(X, False, f[0]), False, w_op, True, M, N, K, f, d=d)
    assert_guard(d, M, N, "forward")
    check(d[:M, :N], X, W, BOUND[fmt], pair_floor(X, W) if pair else 0.0, f"weight forward {fmt}")
    d = guarded(M, K)
    gemm(operand(dY, False, f[0]), False, w_op, False, M, K, N, f, d=d)
    assert_guard(d, M, K, "dgrad")
    check(d[:M, :K], dY, W.t(), BOUND[fmt], pair_floor(dY, W.t()) if pair else 0.0, f"weight dgrad {fmt}")


# ---- 4. long same-sign contractions ----------------------------------------------------------------------------------
# The tensor cores' fp32 accumulation is not round-to-nearest.  On data of one sign its error does not cancel and grows
# with the number of MMAs into one accumulator; promoting the main accumulator every 512 elements bounds that.
SAME_SIGN_BOUND = {"bf16x3": 2.5e-6, "pair0x2": 1.3e-5}   # measured: 6.3e-7 and 3.2e-6, both at K = 32768


@pytest.mark.parametrize("fmt", list(SAME_SIGN_BOUND))
@pytest.mark.parametrize("K", [16384, 32768])
def test_long_same_sign(K, fmt):
    M, N = 256, 256
    f = FMT[fmt]
    g = torch.Generator(device=DEV).manual_seed(K)
    A = torch.rand(M, K, device=DEV, generator=g) * 0.5 + 0.5
    B = torch.rand(K, N, device=DEV, generator=g) * 0.5 + 0.5
    d = guarded(M, N)
    gemm(operand(A, False, f[0]), False, operand(B.t(), True, f[0]), True, M, N, K, f, d=d)
    assert_guard(d, M, N)
    check(d[:M, :N], A, B, SAME_SIGN_BOUND[fmt], 0.0, f"same-sign K={K} {fmt}")


# ---- 5. wide dynamic range -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", ["bf16x3", "pair0x2"])
def test_wide_dynamic_range(fmt):
    """Row and column scales spanning 7 decades (bf16 x 3), or as much of the fp16 range as the pair keeps (below its
    normal range it loses relative precision: the absolute floor)."""
    M, N, K = 200, 264, 1000
    f = FMT[fmt]
    torch.manual_seed(17)
    if fmt == "bf16x3":
        rs, cs = torch.logspace(-4, 3, M, device=DEV), torch.logspace(3, -4, N, device=DEV)
    else:
        rs, cs = torch.logspace(-4, 2, M, device=DEV), torch.logspace(2, -3, N, device=DEV)
    A = torch.randn(M, K, device=DEV) * rs[:, None]
    B = torch.randn(K, N, device=DEV) * cs[None, :]
    d = guarded(M, N)
    gemm(operand(A, False, f[0]), False, operand(B.t(), True, f[0]), True, M, N, K, f, d=d)
    assert_guard(d, M, N)
    check(d[:M, :N], A, B, BOUND[fmt], pair_floor(A, B) if fmt != "bf16x3" else 0.0, f"wide range {fmt}")


# ---- 6. the epilogue matrix ------------------------------------------------------------------------------------------
EPILOGUES = ["none", "bias", "bias_resid", "bias_gelu", "dgelu", "accumulate_alpha", "planes_only"]
PLANE_EPILOGUES = {"bias_gelu", "dgelu", "planes_only"}
# Bounds on an epilogue output's error over its scale (test_epilogue_matrix), worst measured ratio in the comment.
# dGELU's scale adds |A@B| for the fp32 evaluation of gelu'; its measured error is dominated by that term.
EPI_BOUND = {"bf16x3": 8e-7,    # 1.9e-7 (bias + GELU, d)
             "pair0x2": 1.3e-6}  # 3.3e-7 (no epilogue)
DGELU_BOUND = 8e-6               # 2.0e-6 (both formats, d and planes)


def _ulp(x):
    x = x.abs()
    return torch.nextafter(x, torch.full_like(x, float("inf"))) - x


def _readbacks(planes, code, M, N):
    """fp32 values of a guarded plane output, with the absolute floor of each representation."""
    p = planes[:, :M, :N]
    if code == L.PLANES_FP16_PAIR:
        return [("pair", ops.pair_to_float(p), 2 * PAIR_FLOOR)]
    out = [("bf16x3", p[:3].float().sum(0), 0.0)]
    if code == L.PLANES_BF16X3_FP16_PAIR:
        out.append(("pair", ops.planes_to_float(p, fp16=True), 2 * PAIR_FLOOR))
    return out


@pytest.mark.parametrize("fmt", list(STAGE_FMT))
@pytest.mark.parametrize("epi", EPILOGUES)
def test_epilogue_matrix(epi, fmt):
    """Every fused epilogue, on the vectorised path and on the per-element path (forced by ldd % 4 != 0, by a
    misaligned pointer, and by N % 4 != 0), for every output plane-set code.  Values against fp64, the region written
    against a guard band, and the per-element paths against the vectorised one within 2 ulp of fp32."""
    M, K, Nr = 136, 200, 203
    f = STAGE_FMT[fmt]
    torch.manual_seed(EPILOGUES.index(epi) * 10 + len(fmt))
    A, B = torch.randn(M, K, device=DEV), torch.randn(K, Nr, device=DEV) * 0.05
    a_op, b_op = operand(A, False, f[0]), operand(B.t(), True, f[0])
    bias = torch.randn(Nr, device=DEV)
    resid = torch.randn(M, Nr + 5, device=DEV)
    aux_vals = torch.randn(M, Nr, device=DEV) * 2

    def placed(x, shape, shift):
        """``x`` copied into a fresh tensor of ``shape`` whose base is ``shift`` floats past an aligned allocation."""
        t = torch.empty(shift + torch.Size(shape).numel(), device=DEV)[shift:].view(shape)
        t[tuple(slice(0, n) for n in x.shape)] = x
        return t

    acc0 = torch.randn(M, Nr, device=DEV)
    alpha = 0.3 if epi == "accumulate_alpha" else 1.0
    has_d = epi != "planes_only"
    codes = [3, L.PLANES_BF16X3_FP16_PAIR, L.PLANES_FP16_PAIR] if epi in PLANE_EPILOGUES else [None]
    A64, B64 = A.double(), B.double()
    AB, S = A64 @ B64, A64.abs() @ B64.abs()
    bound = DGELU_BOUND if epi == "dgelu" else EPI_BOUND[fmt]
    pair = fmt.startswith("pair")
    for code in codes:
        vec_d = None
        # path: (N, ldd, which pointer is misaligned by one float)
        for path, N, ldd, mis in [("vec", 200, 208, None), ("ldd", 200, 209, None), ("misaligned", 200, 208, True),
                                  ("ragged", Nr, Nr + 13, None)]:
            misal = None
            if mis:
                misal = "bias" if "bias" in epi else ("aux" if epi == "dgelu" else ("d" if has_d else "planes"))
            kw = {}
            if "bias" in epi or epi == "planes_only":
                kw["bias"] = placed(bias[:N], (N,), 1 if misal == "bias" else 0)
            if epi == "bias_resid":
                kw["resid"] = resid
            if epi == "dgelu":
                kw["act"] = L.ACT_DGELU
                kw["aux"] = placed(aux_vals[:, :N], (M, ldd), 1 if misal == "aux" else 0)
            if epi == "bias_gelu":
                kw["act"] = L.ACT_GELU
            d = None
            if has_d:
                if misal == "d":
                    flat = torch.empty((M + 8) * ldd + 1, device=DEV)
                    d = flat[1:].view(M + 8, ldd)
                    d.view(torch.int32).fill_(SENTINEL)
                    if epi == "accumulate_alpha":
                        d[:M, :N] = acc0[:, :N]
                else:
                    d = guarded(M, N, ldd, inner=acc0[:, :N] if epi == "accumulate_alpha" else None)
            planes = None
            if code is not None:
                if misal == "planes":
                    ldp = round8(N) + 8
                    n = L.planes_count(code)
                    flat16 = torch.full((n * (M + 8) * ldp + 2,), NAN16, dtype=torch.int16, device=DEV)
                    planes = flat16[2:].view(n, M + 8, ldp).view(torch.bfloat16)
                else:
                    planes = guarded_planes(code, M, N, ldp=N + 9 if (path == "ldd" and not has_d) else None)
                kw.update(planes_out=planes, planes_code=code)
            gemm(a_op, False, b_op, True, M, N, K, f, d=d, alpha=alpha, accumulate=epi == "accumulate_alpha", **kw)
            what = f"{epi} {fmt} code {code} {path}"
            # fp64 reference of d (value) and of the planes, with the error scale of each
            ab, s = AB[:, :N], S[:, :N]
            val, vs = alpha * ab, alpha * s
            if "bias" in epi or epi == "planes_only":
                b64 = kw["bias"].double()
                val, vs = val + b64, vs + b64.abs()
            if epi == "bias_resid":
                r64 = resid[:, :N].double()
                val, vs = val + r64, vs + r64.abs()
            if epi == "accumulate_alpha":
                a0 = acc0[:, :N].double()
                val, vs = val + a0, vs + a0.abs()
            if epi == "dgelu":
                x = kw["aux"][:, :N].double().requires_grad_(True)
                og.gelu_new(x).sum().backward()
                gp = x.grad.detach()
                val, vs = ab * gp, s * gp.abs() + ab.abs()   # fp32 gelu' is accurate to a few ulp of 1
            pl, ps_ = val, vs
            if epi == "bias_gelu":
                x = val.clone().requires_grad_(True)
                og.gelu_new(x).sum().backward()
                pl = og.gelu_new(val)
                ps_ = vs * x.grad.abs() + val.abs()   # fp32 tanh: a few ulp of 1 times |x|
            floor = pair_floor(A, B[:, :N]) * (alpha if epi != "dgelu" else gp.abs()) if pair else 0.0
            if has_d:
                assert_guard(d, M, N, what)
                check_value(d[:M, :N], val, vs, bound, floor, f"epilogue d {what}")
                if path == "vec":
                    vec_d = d[:M, :N].clone()
                else:
                    got = d[:M, :200]
                    diff = (got - vec_d).abs()
                    bad = int((diff > 2 * _ulp(vec_d)).sum())
                    assert bad == 0, f"{what}: {bad} elements differ from the vectorised path by more than 2 ulp"
            if planes is not None:
                assert_guard(planes, M, N, what)
                for rname, rb, rfloor in _readbacks(planes, code, M, N):
                    check_value(rb, pl, ps_, bound, floor + rfloor * (1 + pl.abs()),
                                f"epilogue planes/{rname} {what}")


# ---- 7. many waves and determinism ---------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", list(STAGE_FMT))
@pytest.mark.parametrize("shape", [(2048, 6400, 1600), (4096, 1600, 6400)], ids=lambda s: "x".join(map(str, s)))
def test_many_waves_deterministic(shape, fmt):
    """800 (and 400) tiles: several waves over 132 SMs with a partial last one.  Two runs agree bit for bit."""
    M, N, K = shape
    f = STAGE_FMT[fmt]
    torch.manual_seed(M + N)
    A, B = torch.randn(M, K, device=DEV), torch.randn(K, N, device=DEV) * 0.05
    a, b = operand(A, False, f[0]), operand(B.t(), True, f[0])
    d1, d2 = guarded(M, N), guarded(M, N)
    gemm(a, False, b, True, M, N, K, f, d=d1)
    gemm(a, False, b, True, M, N, K, f, d=d2)
    assert_guard(d1, M, N)
    check(d1[:M, :N], A, B, BOUND[fmt], pair_floor(A, B) if fmt.startswith("pair") else 0.0, f"waves {fmt}")
    assert torch.equal(d1.view(torch.int32), d2.view(torch.int32)), "two runs of the same GEMM differ"


# ---- 8. argument rejection -------------------------------------------------------------------------------------------
def _raw_gemm(a, a_mn, b, b_mn, M, N, K, nsplit, d=None, ldd=64, **epi):
    e = L.GemmEpilogue()
    e.d, e.ldd, e.alpha = (0 if d is None else d.data_ptr()), ldd, 1.0
    for k, v in epi.items():
        setattr(e, k, v)
    L.call("oob_gemm", C.byref(a), int(a_mn), C.byref(b), int(b_mn), M, N, K, nsplit, C.byref(e), S())


def test_argument_rejection():
    """Each check of oob_gemm, gemm_launch and make_map raises with its message, and nothing is launched."""
    p5 = ops.split(torch.randn(64, 64, device=DEV), nplanes=L.PLANES_BF16X3_FP16_PAIR)
    p2 = ops.split(torch.randn(64, 64, device=DEV), nplanes=2)
    big = torch.zeros(3 * 64 * 72 + 64, dtype=torch.bfloat16, device=DEV)
    d = torch.zeros(64, 64, device=DEV)
    gp = ops.new_planes(64, 64)

    def g(a=p5, b=p5, M=64, N=64, K=64, **kw):
        return lambda: ops.gemm(a, False, b, False, M, N, K, **{"d": d, **kw})

    def raw(desc_a, desc_b=None, M=64, N=64, K=64, nsplit=3, **kw):
        return lambda: _raw_gemm(desc_a, False, desc_b or ops.planes_desc(p5), False, M, N, K, nsplit, d, **kw)

    base = big.data_ptr()
    cases = [
        ("nsplit must be 1..3", g(nsplit=0)),
        ("nsplit must be 1..3", g(nsplit=4)),
        ("empty GEMM", g(M=0)),
        ("empty GEMM", g(K=0)),
        ("mixed fp16 / bf16", g(a_fp16=True, nsplit=2)),
        ("fp16 planes come in pairs", g(a_fp16=True, b_fp16=True, nsplit=3)),
        ("fewer planes than nsplit", g(a=p2, nsplit=3)),
        ("unknown plane-set code 4", g(planes_out=gp, planes_code=4)),
        (r"A \(K-major\) is 64 x 64, need 72 x 64", g(M=72)),
        (r"A \(M-major\) is 64 x 64, need 64 x 72", lambda: ops.gemm(p5, True, p5, False, 72, 64, 64, d=d)),
        (r"B \(K-major\) is 64 x 64, need 72 x 64", g(N=72)),
        (r"B \(N-major\) is 64 x 64, need 64 x 72", lambda: ops.gemm(p5, False, p5, True, 64, 72, 64, d=d)),
        ("strides must be multiples of 8", raw(L.Planes(base, 64, 64, 68, 64 * 72, 3, 0))),
        ("strides must be multiples of 8", raw(L.Planes(base, 64, 64, 64, 64 * 64 + 4, 3, 0))),
        ("must be 16 B aligned", raw(L.Planes(base + 8, 64, 64, 64, 64 * 64, 3, 0))),
        ("cuTensorMapEncodeTiled failed", raw(L.Planes(base, 64, 64, 64, 1 << 40, 3, 0))),
        ("GEMM N = 8388736 too large", raw(ops.planes_desc(p5), L.Planes(base, 8388736, 64, 64, 64 * 64, 3, 0),
                                           N=8388736)),
        ("no output", lambda: _raw_gemm(ops.planes_desc(p5), False, ops.planes_desc(p5), False, 64, 64, 64, 3)),
        ("accumulate needs d", lambda: _raw_gemm(ops.planes_desc(p5), False, ops.planes_desc(p5), False, 64, 64, 64,
                                                 3, planes=gp.data_ptr(), ldp=64, plane_stride=64 * 64,
                                                 nplanes_out=3, accumulate=1)),
        ("dGELU needs aux", g(act=L.ACT_DGELU)),
    ]
    lib = L.load()
    torch.cuda.synchronize()
    n0 = lib.oob_launch_count()
    for msg, fn in cases:
        with pytest.raises(L.OobleckB200Error, match=msg):
            fn()
    assert lib.oob_launch_count() == n0, "a rejected GEMM was launched"
    torch.cuda.synchronize()
    assert d.abs().sum() == 0 and torch.isfinite(d).all()


# ---- 9. tensor-map cache eviction ----------------------------------------------------------------------------------
def test_tensor_map_cache_eviction():
    """The TMA descriptor cache (gemm.cu) is cleared when it holds 16384 maps.  Each call below reads one fixed A and a
    B that slides 8 elements further through a large buffer: A's lookup hits, B's misses.  So every clear falls on B's
    lookup, after A's map was found, and the call after a clear misses A as well (two misses instead of one).  Every
    result is compared with fp64 at the end."""
    n = 17000
    torch.manual_seed(19)
    A = torch.randn(64, 64, device=DEV)
    a = ops.split(A)
    src = torch.randn(64 * 64 + 8 * n, device=DEV)
    flat = torch.empty(3, src.numel(), dtype=torch.bfloat16, device=DEV)
    L.call("oob_split_planes", P(src), P(flat), src.numel(), flat.stride(0), 3, S())
    out = torch.full((n, 64, 64), float("nan"), device=DEV)
    lib = L.load()
    e0 = lib.oob_tensor_map_encodes()
    misses = []
    for i in range(n):
        b = flat.as_strided((3, 64, 64), (flat.stride(0), 64, 1), 8 * i)
        before = lib.oob_tensor_map_encodes()
        ops.gemm(a, False, b, False, 64, 64, 64, d=out[i])
        misses.append(lib.oob_tensor_map_encodes() - before)
    total = lib.oob_tensor_map_encodes() - e0
    assert total > 16384, total
    cleared_on_b = [i - 1 for i in range(1, n) if misses[i] == 2]
    assert cleared_on_b, "no cache clear observed"
    Bw = src.as_strided((n, 64, 64), (8, 64, 1)).double()      # B_i stored [N][K]
    A64 = A.double()
    check_value(out, A64 @ Bw.transpose(1, 2), A64.abs() @ Bw.abs().transpose(1, 2), BOUND["bf16x3"], 0.0,
                f"cache eviction ({len(cleared_on_b)} clears)")
