"""GPU parity tests of every CUDA kernel, through the C ABI, against plain torch (fp64 / fp32 references)."""
import ctypes as C
import math

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]

if not torch.cuda.is_available():  # collected on CPU, skipped (never run without -m gpu anyway)
    pytest.skip("needs CUDA", allow_module_level=True)

from oobleck_b200 import lib as L  # noqa: E402
from oobleck_b200 import ops  # noqa: E402
from oracle import gpt2 as og  # noqa: E402

DEV = "cuda"


def P(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def S():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def rel_err(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


def test_split_roundtrip():
    x = torch.randn(1000, 72, device=DEV) * torch.logspace(-6, 6, 72, device=DEV)
    p = ops.split(x)
    back = ops.planes_to_float(p)
    assert rel_err(back, x) < 1e-7
    assert ((back - x).abs() <= x.abs() * 2 ** -22).all()


def test_split5_fp16_pair():
    """5-plane buffers: planes 0-2 = bf16 x 3 (24 bits, any range), planes 3-4 = fp16 pair (22 bits, |x| < 65504)."""
    x = torch.randn(1000, 72, device=DEV) * torch.logspace(-3, 3, 72, device=DEV)
    p = ops.split(x, nplanes=5)
    assert rel_err(ops.planes_to_float(p), x) < 1e-7
    back = ops.planes_to_float(p, fp16=True)
    assert ((back - x).abs() <= x.abs() * 2 ** -21 + 2 ** -35).all()   # 22 bits, absolute floor 2^-36
    # saturation instead of inf, and graceful loss of precision below the fp16 normal range
    y = torch.tensor([[1e6, -1e6, 1e-7, 3e-9, 0.0, 65504.0, 1.0, -2.5]], device=DEV)
    q = ops.planes_to_float(ops.split(y, nplanes=5), fp16=True)
    assert torch.isfinite(q).all() and abs(q[0, 0].item() - 65504.0 - 65504.0 / 2048) < 1 and q[0, 4] == 0
    assert abs(q[0, 2].item() - 1e-7) < 2 ** -35 and q[0, 6] == 1.0 and q[0, 7] == -2.5


@pytest.mark.parametrize("a_mn", [False, True])
@pytest.mark.parametrize("b_mn", [False, True])
@pytest.mark.parametrize("shape", [(256, 384, 512), (304, 200, 136), (2048, 512, 1600), (256, 128, 6400)])
def test_gemm_fp16_pair(a_mn, b_mn, shape):
    """fp16 x 2 operands: 3 tensor-core products must stay fp32-grade (same bar as the 6-product bf16 x 3 mode)."""
    M, N, K = shape
    torch.manual_seed(M + N + K)
    A = torch.randn(M, K, device=DEV)
    B = torch.randn(K, N, device=DEV) * 0.02
    ap = ops.split(A.t().contiguous() if a_mn else A, nplanes=5)
    bp = ops.split(B if b_mn else B.t().contiguous(), nplanes=5)
    ref = A.double() @ B.double()
    d = torch.full((M, N), float("nan"), device=DEV)
    ops.gemm(ap, a_mn, bp, b_mn, M, N, K, nsplit=2, d=d, a_fp16=True, b_fp16=True)
    err = rel_err(d, ref)
    d3 = torch.empty_like(d)
    ops.gemm(ap, a_mn, bp, b_mn, M, N, K, nsplit=3, d=d3)
    print(f"fp16x2 err {err:.2e}   bf16x3 err {rel_err(d3, ref):.2e}")
    # 22-bit operands: max-normalised error a few 1e-7 (the 24-bit bf16 x 3 mode: ~2e-7); parity budget is 1e-4
    assert err < 3e-6, err
    # one plane only = plain fp16 GEMM
    ops.gemm(ap, a_mn, bp, b_mn, M, N, K, nsplit=1, d=d, a_fp16=True, b_fp16=True)
    assert rel_err(d, ref) < 3e-3


def test_gemm_epilogue_five_planes():
    M, N, K = 256, 384, 320
    A, W = torch.randn(M, K, device=DEV), torch.randn(K, N, device=DEV) * 0.05
    bias = torch.randn(N, device=DEV)
    ap, wp = ops.split(A, nplanes=5), ops.split(W, nplanes=5)
    pre_ref = A.double() @ W.double() + bias.double()
    d = torch.empty(M, N, device=DEV)
    gp = ops.new_planes(M, N, 5)
    ops.gemm(ap, False, wp, True, M, N, K, nsplit=2, d=d, bias=bias, act=L.ACT_GELU, planes_out=gp, a_fp16=True,
             b_fp16=True)
    assert rel_err(d, pre_ref) < 2e-6
    assert rel_err(ops.planes_to_float(gp), og.gelu_new(pre_ref)) < 2e-6
    assert rel_err(ops.planes_to_float(gp, fp16=True), og.gelu_new(pre_ref)) < 2e-6


@pytest.mark.parametrize("a_mn", [False, True])
@pytest.mark.parametrize("b_mn", [False, True])
@pytest.mark.parametrize("shape", [(128, 128, 64), (256, 384, 512), (304, 200, 136), (1024, 768, 768), (256, 128, 6400)])
def test_gemm_majors(a_mn, b_mn, shape):
    M, N, K = shape
    A = torch.randn(M, K, device=DEV)
    B = torch.randn(K, N, device=DEV)
    ap = ops.split(A.t().contiguous() if a_mn else A)
    bp = ops.split(B if b_mn else B.t().contiguous())
    ref = A.double() @ B.double()
    tol = {1: 2e-2, 2: 1e-4, 3: 1e-6}
    for ns in (3, 2, 1):
        d = torch.full((M, N), float("nan"), device=DEV)
        ops.gemm(ap, a_mn, bp, b_mn, M, N, K, nsplit=ns, d=d)
        err = rel_err(d, ref)
        assert err < tol[ns], (ns, err)


def test_gemm_epilogues():
    M, N, K = 384, 256, 320
    A, W = torch.randn(M, K, device=DEV), torch.randn(K, N, device=DEV) * 0.05
    bias, R = torch.randn(N, device=DEV), torch.randn(M, N, device=DEV)
    ap, wp = ops.split(A), ops.split(W)
    pre_ref = A.double() @ W.double() + bias.double()
    # bias + residual
    d = torch.empty(M, N, device=DEV)
    ops.gemm(ap, False, wp, True, M, N, K, d=d, bias=bias, resid=R)
    assert rel_err(d, pre_ref + R.double()) < 2e-6
    # bias + GELU: d = pre-activation, planes = gelu(pre)
    gp = ops.new_planes(M, N)
    ops.gemm(ap, False, wp, True, M, N, K, d=d, bias=bias, act=L.ACT_GELU, planes_out=gp)
    assert rel_err(d, pre_ref) < 2e-6
    assert rel_err(ops.planes_to_float(gp), og.gelu_new(pre_ref)) < 2e-6
    # accumulate (wgrad): d += A^T-major product
    X, dY = torch.randn(M, K, device=DEV), torch.randn(M, N, device=DEV)
    acc = torch.randn(K, N, device=DEV)
    want = acc.double() + X.double().t() @ dY.double()
    ops.gemm(ops.split(X), True, ops.split(dY), True, K, N, M, d=acc, accumulate=True)
    assert rel_err(acc, want) < 2e-6
    # dGELU epilogue: planes = (dY W^T) * gelu'(pre)
    pre = torch.randn(M, K, device=DEV)
    pre64 = pre.double().requires_grad_(True)
    og.gelu_new(pre64).backward((dY.double() @ W.double().t()))
    out = ops.new_planes(M, K)
    d2 = torch.empty(M, K, device=DEV)
    ops.gemm(ops.split(dY), False, wp, False, M, K, N, d=d2, act=L.ACT_DGELU, aux=pre, planes_out=out)
    assert rel_err(d2, pre64.grad) < 5e-6
    assert rel_err(ops.planes_to_float(out), pre64.grad) < 5e-6


@pytest.mark.parametrize("E", [64, 768, 1600])
def test_layernorm_fwd_bwd(E):
    rows = 515
    x = torch.randn(rows, E, device=DEV) * 2 + 0.5
    g, b = torch.randn(E, device=DEV), torch.randn(E, device=DEV)
    y = torch.empty_like(x)
    yp = ops.new_planes(rows, E)
    mean, rstd = torch.empty(rows, device=DEV), torch.empty(rows, device=DEV)
    L.call("oob_layernorm_fwd", P(x), P(g), P(b), P(y), P(yp), yp.stride(0), 3, P(mean), P(rstd), rows, E, 1e-5, S())
    x64 = x.double().requires_grad_(True)
    g64, b64 = g.double().requires_grad_(True), b.double().requires_grad_(True)
    ref = torch.nn.functional.layer_norm(x64, (E,), g64, b64, 1e-5)
    assert rel_err(y, ref) < 2e-6
    assert rel_err(ops.planes_to_float(yp), ref) < 2e-6
    dy, dres = torch.randn(rows, E, device=DEV), torch.randn(rows, E, device=DEV)
    ref.backward(dy.double())
    dx = torch.empty_like(x)
    dxp = ops.new_planes(rows, E)
    dg, db = torch.ones(E, device=DEV), torch.ones(E, device=DEV)  # accumulate onto ones
    part = torch.empty(L.load().oob_ln_bwd_partials_floats(E), device=DEV)
    L.call("oob_layernorm_bwd", P(dy), P(x), P(mean), P(rstd), P(g), P(dres), P(dx), P(dxp), dxp.stride(0), 3, P(dg),
           P(db), P(part), rows, E, 1.0, S())
    assert rel_err(dx, x64.grad + dres.double()) < 5e-6
    assert rel_err(ops.planes_to_float(dxp), x64.grad + dres.double()) < 5e-6
    assert rel_err(dg - 1, g64.grad) < 5e-6
    assert rel_err(db - 1, b64.grad) < 5e-6
    # loss-scaled gradient in, fp16 pair out, parameter gradients unscaled
    S_ = 4096.0
    dg2, db2 = torch.zeros(E, device=DEV), torch.zeros(E, device=DEV)
    dys, drs = dy * S_, dres * S_
    L.call("oob_layernorm_bwd", P(dys), P(x), P(mean), P(rstd), P(g), P(drs), P(dx), P(dxp), dxp.stride(0),
           ops.PLANES_FP16_PAIR, P(dg2), P(db2), P(part), rows, E, 1.0 / S_, S())
    assert rel_err(dx / S_, x64.grad + dres.double()) < 5e-6
    assert rel_err(ops.pair_to_float(dxp) / S_, x64.grad + dres.double()) < 5e-6
    assert rel_err(dg2, g64.grad) < 5e-6 and rel_err(db2, b64.grad) < 5e-6


def test_colsum():
    a = torch.randn(1000, 4800, device=DEV)
    out = torch.ones(4800, device=DEV)
    part = torch.empty(L.load().oob_colsum_partials_floats(4800), device=DEV)
    L.call("oob_colsum_accumulate", P(a), a.stride(0), 1000, 4800, P(out), P(part), 1.0, S())
    assert rel_err(out - 1, a.double().sum(0)) < 2e-6


def ref_attention(qkv, B, T, H, D):
    E = H * D
    q, k, v = qkv.view(B, T, 3 * E).split(E, dim=2)
    q, k, v = (t.view(B, T, H, D).transpose(1, 2) for t in (q, k, v))
    att = (q @ k.transpose(-1, -2)) / math.sqrt(D)
    mask = torch.tril(torch.ones(T, T, dtype=torch.bool, device=qkv.device))
    att = att.masked_fill(~mask, float("-inf")).softmax(-1)
    return (att @ v).transpose(1, 2).reshape(B * T, E)


@pytest.mark.parametrize("h2", [0, 1])
@pytest.mark.parametrize("B,T,H", [(2, 128, 3), (1, 100, 2), (3, 64, 2), (1, 192, 1), (2, 333, 2), (2, 1024, 4),
                                   (2, 1024, 25)])
def test_attention_fwd_bwd(B, T, H, h2):
    """h2 = 1: q|k|v and dO as fp16 pairs (3 products per MAC), dO additionally loss-scaled like in the stage."""
    D, E = 64, H * 64
    torch.manual_seed(B * 1000 + T + H)
    qkv = torch.randn(B * T, 3 * E, device=DEV)
    out = torch.empty(B * T, E, device=DEV)
    outp = ops.new_planes(B * T, E)
    lse = torch.empty(B, H, T, device=DEV)
    code = ops.PLANES_FP16_PAIR if h2 else 3
    gscale = 256.0 if h2 else 1.0
    qp = ops.split(qkv, nplanes=code)
    L.call("oob_attention_fwd", P(qp), qp.stride(0), h2, P(out), P(outp), outp.stride(0), 3, P(lse), B, T, H, D, S())
    q64 = qkv.double().requires_grad_(True)
    ref = ref_attention(q64, B, T, H, D)
    assert rel_err(out, ref) < 5e-6
    assert rel_err(ops.planes_to_float(outp), ref) < 5e-6
    dout = torch.randn(B * T, E, device=DEV)
    ref.backward(dout.double())
    dqkv = torch.full((B * T, 3 * E), float("nan"), device=DEV)
    dqp = ops.new_planes(B * T, 3 * E)
    delta = torch.empty(B, H, T, device=DEV)
    dout_s = dout * gscale
    dop = ops.split(dout_s, nplanes=code)
    L.call("oob_attention_bwd", P(qp), qp.stride(0), h2, P(out), P(dout_s), P(dop), dop.stride(0), P(lse), P(delta),
           P(dqkv), P(dqp), dqp.stride(0), code, B, T, H, D, S())
    assert rel_err(dqkv / gscale, q64.grad) < 1e-5
    got = ops.pair_to_float(dqp) if h2 else ops.planes_to_float(dqp)
    assert rel_err(got / gscale, q64.grad) < 1e-5


def test_attention_lazy_rescale_and_wide_scores():
    """The forward keeps O in registers and moves a row's softmax reference point only when its maximum has grown by
    more than 2^8 (attention_sm90.cu).  Keys whose norm grows along the sequence force that rescale path many times per
    row; scores spanning +-60 also exercise the exponent range of the fp16-pair probabilities."""
    B, T, H, D = 2, 512, 2, 64
    E = H * D
    torch.manual_seed(5)
    qkv = torch.randn(B * T, 3 * E, device=DEV)
    ramp = torch.linspace(0.2, 6.0, T, device=DEV).repeat(B).unsqueeze(1)
    qkv[:, E:2 * E] *= ramp                       # |k_t| grows with t: the running maximum keeps jumping
    qkv[:, :E] *= 1.5
    for h2 in (1, 0):
        code = ops.PLANES_FP16_PAIR if h2 else 3
        qp = ops.split(qkv, nplanes=code)
        out = torch.empty(B * T, E, device=DEV)
        outp = ops.new_planes(B * T, E)
        lse = torch.empty(B, H, T, device=DEV)
        L.call("oob_attention_fwd", P(qp), qp.stride(0), h2, P(out), P(outp), outp.stride(0), 3, P(lse), B, T, H, D, S())
        q64 = qkv.double().requires_grad_(True)
        ref = ref_attention(q64, B, T, H, D)
        assert rel_err(out, ref) < 5e-6, (h2, rel_err(out, ref))
        q, k, _ = q64.detach().view(B, T, 3 * E).split(E, dim=2)
        sc = (q.view(B, T, H, D).transpose(1, 2) @ k.view(B, T, H, D).transpose(1, 2).transpose(-1, -2)) / 8.0
        sc = sc.masked_fill(~torch.tril(torch.ones(T, T, dtype=torch.bool, device=DEV)), float("-inf"))
        assert rel_err(lse, torch.logsumexp(sc, -1)) < 2e-6
        dout = torch.randn(B * T, E, device=DEV)
        ref.backward(dout.double())
        dqkv = torch.full((B * T, 3 * E), float("nan"), device=DEV)
        dqp = ops.new_planes(B * T, 3 * E)
        delta = torch.empty(B, H, T, device=DEV)
        gs = 64.0 if h2 else 1.0
        dop = ops.split(dout * gs, nplanes=code)
        L.call("oob_attention_bwd", P(qp), qp.stride(0), h2, P(out), P(dout * gs), P(dop), dop.stride(0), P(lse), P(delta),
               P(dqkv), P(dqp), dqp.stride(0), code, B, T, H, D, S())
        assert rel_err(dqkv / gs, q64.grad) < 1e-5, (h2, rel_err(dqkv / gs, q64.grad))


def test_embedding_fwd_bwd():
    B, T, E, V = 2, 64, 128, 1000
    ids = torch.randint(0, V, (B, T), device=DEV)
    ids[0, :8] = 7  # repeated tokens exercise the scatter-add
    wte, wpe = torch.randn(V, E, device=DEV), torch.randn(T, E, device=DEV)
    h = torch.empty(B * T, E, device=DEV)
    L.call("oob_embedding_fwd", P(ids), P(wte), P(wpe), P(h), B * T, T, E, S())
    ref = wte[ids].view(B * T, E) + wpe.repeat(B, 1)
    assert torch.equal(h, ref)
    dh = torch.randn(B * T, E, device=DEV)
    dwte, dwpe = torch.zeros_like(wte), torch.zeros_like(wpe)
    L.call("oob_embedding_bwd", P(ids), P(dh), P(dwte), P(dwpe), B, T, E, 1.0, S())
    want_wte = torch.zeros_like(wte).double().index_add_(0, ids.view(-1), dh.double())
    assert rel_err(dwte, want_wte) < 2e-6
    assert rel_err(dwpe, dh.double().view(B, T, E).sum(0)) < 2e-6


def test_cross_entropy():
    B, T, V = 2, 33, 50257
    Vp = (V + 63) // 64 * 64
    logits = torch.randn(B * T, Vp, device=DEV) * 3
    labels = torch.randint(0, V, (B, T), device=DEV)
    row_loss = torch.empty(B * T, device=DEV)
    loss, total = torch.zeros(1, device=DEV), torch.ones(1, device=DEV)
    dp = ops.new_planes(B * T, Vp)
    L.call("oob_cross_entropy", P(logits), Vp, P(labels), B, T, V, P(row_loss), P(loss), P(total), P(dp), Vp,
           dp.stride(0), 3, 1.0, S())
    l64 = logits[:, :V].double().view(B, T, V).requires_grad_(True)
    ref = torch.nn.functional.cross_entropy(l64[:, :-1].reshape(-1, V), labels[:, 1:].reshape(-1))
    ref.backward()
    assert abs(loss.item() - ref.item()) < 1e-5 * abs(ref.item())
    assert abs(total.item() - 1 - ref.item()) < 1e-5 * abs(ref.item())
    got = ops.planes_to_float(dp)
    assert rel_err(got[:, :V], l64.grad.view(B * T, V)) < 5e-6
    assert (got[:, V:] == 0).all()
    # loss-scaled fp16-pair gradient
    L.call("oob_cross_entropy", P(logits), Vp, P(labels), B, T, V, P(row_loss), P(loss), P(total), P(dp), Vp,
           dp.stride(0), ops.PLANES_FP16_PAIR, 1024.0, S())
    got = ops.pair_to_float(dp) / 1024.0
    assert rel_err(got[:, :V], l64.grad.view(B * T, V)) < 5e-6
    assert (got[:, V:] == 0).all()


def test_cross_entropy_ignored_labels():
    """HF GPT-2's loss is CrossEntropyLoss(ignore_index=-100, mean over the targets that count): padded labels (and ids
    outside the vocabulary) give no loss, no gradient, and do not enter the divisor."""
    B, T, V = 3, 17, 1000
    Vp = (V + 63) // 64 * 64
    torch.manual_seed(1)
    logits = torch.randn(B * T, Vp, device=DEV) * 2
    labels = torch.randint(0, V, (B, T), device=DEV)
    labels[0, 5:9] = -100
    labels[2, 1] = -100
    labels[1, 16] = V + 7            # out of range: ignored, never dereferenced
    row_loss = torch.empty(B * T, device=DEV)
    loss, total = torch.zeros(1, device=DEV), torch.zeros(1, device=DEV)
    dp = ops.new_planes(B * T, Vp)
    L.call("oob_cross_entropy", P(logits), Vp, P(labels), B, T, V, P(row_loss), P(loss), P(total), P(dp), Vp,
           dp.stride(0), 3, 1.0, S())
    l64 = logits[:, :V].double().view(B, T, V).requires_grad_(True)
    tgt = labels[:, 1:].clone()
    tgt[tgt >= V] = -100
    ref = torch.nn.functional.cross_entropy(l64[:, :-1].reshape(-1, V), tgt.reshape(-1), ignore_index=-100)
    ref.backward()
    assert abs(loss.item() - ref.item()) < 1e-5 * abs(ref.item())
    got = ops.planes_to_float(dp)
    assert rel_err(got[:, :V], l64.grad.view(B * T, V)) < 5e-6
    ignored = (tgt.reshape(-1) == -100)
    rows = torch.arange(B * T, device=DEV).view(B, T)[:, :-1].reshape(-1)[ignored]
    assert (got[rows] == 0).all() and (row_loss[rows] == 0).all()


def test_adamw_matches_torch():
    n = 100003
    p0, g = torch.randn(n, device=DEV), torch.randn(n, device=DEV)
    p_ref = torch.nn.Parameter(p0.clone())
    opt = torch.optim.AdamW([p_ref], lr=1e-3, betas=(0.9, 0.999), eps=1e-8, fused=True)
    p, m, v = p0.clone(), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    ps = (n + 7) // 8 * 8
    planes = torch.empty(3, ps, dtype=torch.bfloat16, device=DEV)
    for step in range(1, 4):
        gs = g * step
        p_ref.grad = gs.clone()
        opt.step()
        L.call("oob_adamw_step", P(p), P(gs), P(m), P(v), P(planes), ps, 3, n, 1e-3, 0.9, 0.999, 1e-8, 0.01, step, S())
        assert rel_err(p, p_ref.data) < 1e-6
    assert rel_err(planes[:, :n].float().sum(0), p) < 1e-7
