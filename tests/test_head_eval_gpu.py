"""The forward-only LM head ``oob_head_eval``: ln_f, the LM-head GEMM with the row log-sum-exp epilogue and the merge of
its partials, checked against float64 cross entropy on the same split planes, against the materialising
``oob_head_forward`` and for its argument checks.  GPT-2's vocabulary (V = 50257, logits row stride 50304), so the
last 128-column tile is ragged."""
import ctypes as C
import math

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

if not torch.cuda.is_available():
    pytest.skip("needs CUDA", allow_module_level=True)

from oobleck_b200 import lib as L  # noqa: E402
from oobleck_b200.lib import OobDims, OobHeadCtx, OobLayerParams  # noqa: E402

E, V, VP = 1600, 50257, 50304
NT = (V + 127) // 128
SENTINEL = 0x7FC0DEAD   # a NaN pattern no kernel writes

# Operand formats of the head: (fwd_fp16, bwd_fp16, nsplit, weight plane-set code, ln_f plane-set code of the eval)
FORMATS = {
    "fp16pair_pair_only": (1, 1, 3, L.PLANES_FP16_PAIR, L.PLANES_FP16_PAIR),
    "fp16pair_5planes": (1, 0, 3, L.PLANES_BF16X3_FP16_PAIR, L.PLANES_FP16_PAIR),
    "fp16pair_5planes_lnf5": (1, 0, 3, L.PLANES_BF16X3_FP16_PAIR, L.PLANES_BF16X3_FP16_PAIR),
    "bf16x3": (0, 0, 3, 3, 3),
    "bf16_nsplit2": (0, 0, 2, 3, 2),
    "bf16_nsplit1": (0, 0, 1, 3, 1),
}
SHAPES = [(2, 1024), (500, 2)]    # M = 2048; M = 1000 with T = 2 (one target per sequence)

# Bounds, about 4x the worst figure measured on one NVIDIA H100 80GB HBM3 (700 W power limit) over every format and
# shape above.  Per row: |eval - fp64| / (1 + |fp64|) and |eval - oob_head_forward| / (1 + |forward|).
FP64_BOUND = 8e-6           # measured 2.1e-6 (bf16 planes, nsplit 2); 4.0e-7 for the fp16 pairs
FORWARD_BOUND = 8e-7        # measured 1.9e-7: both read bitwise-identical logits, only the summation order differs


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return C.c_void_p(t.data_ptr())


def _round8(n):
    return (n + 7) // 8 * 8


class Head:
    """Head parameters as a stage holds them: flat fp32 [ln_f.w, ln_f.b, W (V x E)] and their planes."""

    def __init__(self, fmt, B, T, seed=0):
        self.fwd_fp16, self.bwd_fp16, self.nsplit, self.wcode, self.lnf_code = FORMATS[fmt]
        self.B, self.T, self.M = B, T, B * T
        g = torch.Generator(device="cuda").manual_seed(seed)
        n = 2 * E + V * E
        self.w = torch.empty(n, device="cuda")
        self.w[:E] = 1.0 + 0.1 * torch.randn(E, device="cuda", generator=g)
        self.w[E:2 * E] = 0.05 * torch.randn(E, device="cuda", generator=g)
        self.w[2 * E:] = 0.05 * torch.randn(V * E, device="cuda", generator=g)
        self.ps = _round8(n)
        self.planes = torch.empty(L.planes_count(self.wcode), self.ps, dtype=torch.bfloat16, device="cuda")
        L.call("oob_split_planes", _p(self.w), _p(self.planes), n, self.ps, self.wcode, _stream())
        self.grad = torch.zeros(n, device="cuda")
        self.params = OobLayerParams(self.w.data_ptr(), self.planes.data_ptr(), self.ps, self.grad.data_ptr())
        self.x = torch.randn(self.M, E, device="cuda", generator=g)
        lab = torch.randint(0, V, (B, T), device="cuda", generator=g)
        flat = lab.view(-1)
        flat[::7] = -100                     # HF's ignore_index
        flat[3::11] = V                      # out of range: ignored too
        flat[5::13] = V - 1                  # the ragged last tile
        flat[6::17] = 0
        self.labels = lab.contiguous()
        self.dims = OobDims(B, T, E, E // 64, V, VP, 1e-5, self.nsplit, self.fwd_fp16, self.bwd_fp16, 1024.0)


class EvalBuffers:
    GUARD = 64   # floats of sentinel on either side of the partials and the row losses

    def __init__(self, h: Head):
        M, G = h.M, self.GUARD
        self.lnf = torch.empty(L.planes_count(h.lnf_code), M, E, dtype=torch.bfloat16, device="cuda")
        self.mean = torch.empty(M, device="cuda")
        self.rstd = torch.empty(M, device="cuda")
        npart = L.load().oob_head_eval_partials_floats(M, V)
        assert npart == 2 * M * NT
        self.part_raw = torch.full((npart + 2 * G,), SENTINEL, dtype=torch.int32, device="cuda")
        self.part = self.part_raw[G:G + npart].view(torch.float32)
        self.row_raw = torch.full((M + 2 * G,), SENTINEL, dtype=torch.int32, device="cuda")
        self.row_loss = self.row_raw[G:G + M].view(torch.float32)
        self.loss = torch.zeros(1, device="cuda")
        self.acc = torch.zeros(2, dtype=torch.float64, device="cuda")

    def guards_intact(self):
        G = self.GUARD
        return all(bool((t[:G] == SENTINEL).all()) and bool((t[-G:] == SENTINEL).all())
                   for t in (self.part_raw, self.row_raw))


def run_eval(h: Head, b: EvalBuffers, lnf_code=None, partials=None, dims=None, acc=True):
    return L.load().oob_head_eval(C.byref(dims or h.dims), C.byref(h.params), _p(h.x), _p(h.labels), _p(b.lnf),
                                  h.lnf_code if lnf_code is None else lnf_code, _p(b.mean), _p(b.rstd),
                                  C.c_void_p(partials if partials is not None else b.part.data_ptr()),
                                  _p(b.row_loss), _p(b.loss), _p(b.acc) if acc else None, _stream())


def planes_value(planes, code, nsplit, fwd_fp16):
    """float64 value of what a forward GEMM reads of a plane buffer written with ``code``."""
    if fwd_fp16:
        pair = planes[0:2] if code == L.PLANES_FP16_PAIR else planes[3:5]
        h = pair.view(torch.float16).double()
        return h[0] + h[1] / 2048.0
    return planes[:nsplit].double().sum(0)


def fp64_row_loss(h: Head, b: EvalBuffers):
    a = planes_value(b.lnf, h.lnf_code, h.nsplit, h.fwd_fp16)                             # [M, E]
    wp = h.planes[:, 2 * E:2 * E + V * E].view(-1, V, E)
    w = planes_value(wp, h.wcode, h.nsplit, h.fwd_fp16)                                    # [V, E]
    logits = a @ w.t()
    del a, w
    lse = torch.logsumexp(logits, dim=1)
    t = torch.arange(h.M, device="cuda") % h.T
    tgt = torch.full((h.M,), -1, dtype=torch.int64, device="cuda")
    flat = h.labels.view(-1)
    tgt[:-1] = flat[1:]
    valid = (t < h.T - 1) & (tgt >= 0) & (tgt < V)
    picked = logits.gather(1, tgt.clamp(0, V - 1).view(-1, 1)).view(-1)
    return torch.where(valid, lse - picked, torch.zeros_like(lse)), valid


def forward_row_loss(h: Head):
    M = h.M
    lnf_code = {(1, 1): L.PLANES_FP16_PAIR, (1, 0): L.PLANES_BF16X3_FP16_PAIR}.get((h.fwd_fp16, h.bwd_fp16), 3)
    t = {"lnf_planes": torch.empty(L.planes_count(lnf_code), M, E, dtype=torch.bfloat16, device="cuda"),
         "mean": torch.empty(M, device="cuda"), "rstd": torch.empty(M, device="cuda"),
         "logits": torch.empty(M, VP, device="cuda"),
         "dlogits_planes": torch.empty(3, M, VP, dtype=torch.bfloat16, device="cuda"),
         "row_loss": torch.empty(M, device="cuda"), "loss": torch.zeros(1, device="cuda")}
    ctx = OobHeadCtx(**{k: v.data_ptr() for k, v in t.items()})
    L.call("oob_head_forward", C.byref(h.dims), C.byref(h.params), _p(h.x), _p(h.labels), C.byref(ctx), None,
           _stream())
    return t["row_loss"].clone(), float(t["loss"])


@pytest.mark.parametrize("B,T", SHAPES)
@pytest.mark.parametrize("fmt", list(FORMATS))
def test_head_eval_matches_fp64_and_forward(fmt, B, T):
    h = Head(fmt, B, T)
    b = EvalBuffers(h)
    L.check(run_eval(h, b), "oob_head_eval")
    torch.cuda.synchronize()
    assert b.guards_intact(), "a write outside the partial buffer or the row losses"
    got = b.row_loss.double()
    assert bool(torch.isfinite(got).all())

    want, valid = fp64_row_loss(h, b)
    assert bool((got[~valid] == 0).all()), "rows without a target must contribute nothing"
    r64 = float(((got - want).abs() / (1 + want.abs())).max())

    fwd_rows, fwd_loss = forward_row_loss(h)
    rf = float(((got - fwd_rows.double()).abs() / (1 + fwd_rows.double().abs())).max())
    n = int(valid.sum())
    mean = float(got.sum()) / max(n, 1)
    print(f"{fmt} M={h.M}: |eval - fp64| ratio {r64:.2e}, |eval - forward| ratio {rf:.2e}, loss {float(b.loss):.7f} "
          f"forward {fwd_loss:.7f}, targets {n}")
    assert r64 <= FP64_BOUND, (r64, FP64_BOUND)
    assert rf <= FORWARD_BOUND, (rf, FORWARD_BOUND)
    assert math.isclose(float(b.loss), mean, rel_tol=1e-5)
    assert math.isclose(float(b.loss), fwd_loss, rel_tol=1e-5)
    # the accumulator: the micro-batch mean and the number of targets counted
    assert float(b.acc[0]) == float(b.loss[0]) and int(b.acc[1]) == n
    L.check(run_eval(h, b), "oob_head_eval")
    torch.cuda.synchronize()
    assert float(b.acc[0]) == 2 * float(b.loss[0]) and int(b.acc[1]) == 2 * n


@pytest.mark.parametrize("fmt", ["fp16pair_pair_only", "bf16x3"])
def test_head_eval_bit_identical_run_to_run(fmt):
    h = Head(fmt, 2, 1024, seed=3)
    b = EvalBuffers(h)
    outs = []
    for _ in range(3):
        b.part.zero_()
        b.row_loss.zero_()
        L.check(run_eval(h, b, acc=False), "oob_head_eval")
        torch.cuda.synchronize()
        outs.append((b.part.clone(), b.row_loss.clone(), b.loss.clone()))
    for o in outs[1:]:
        for x, y in zip(outs[0], o):
            assert torch.equal(x.view(torch.int32), y.view(torch.int32))
    assert float(b.acc[0]) == 0 and float(b.acc[1]) == 0, "acc = NULL: nothing accumulated"


def test_head_eval_argument_checks_launch_nothing():
    h = Head("fp16pair_pair_only", 1, 256, seed=5)
    b = EvalBuffers(h)
    lib = L.load()
    bad_vp = OobDims(1, 256, E, E // 64, V, V, 1e-5, 3, 1, 1, 1024.0)
    short_t = OobDims(128, 1, E, E // 64, V, VP, 1e-5, 3, 1, 1, 1024.0)
    bf16_dims = OobDims(1, 256, E, E // 64, V, VP, 1e-5, 3, 0, 0, 1.0)
    cases = [
        (dict(lnf_code=4), "unknown plane-set code 4"),
        (dict(lnf_code=7), "unknown plane-set code 7"),
        (dict(lnf_code=3), "fwd_fp16 reads the fp16 pair"),
        (dict(lnf_code=2, dims=bf16_dims), "fewer than nsplit"),
        (dict(partials=b.part.data_ptr() + 4), "partial buffer must be 8 B aligned"),
        (dict(dims=short_t), "bad micro-batch shape"),
        (dict(dims=bad_vp), "vocab_padded must be a multiple of 64"),
    ]
    torch.cuda.synchronize()
    for kw, msg in cases:
        before = lib.oob_launch_count()
        rc = run_eval(h, b, **kw)
        assert rc != 0, kw
        assert msg in lib.oob_last_error().decode(), (kw, lib.oob_last_error())
        assert lib.oob_launch_count() == before, f"{kw}: a kernel was launched"
    torch.cuda.synchronize()
    assert b.guards_intact()
    assert bool((b.row_raw == SENTINEL).all()), "a failed call wrote row losses"
