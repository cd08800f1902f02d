"""Single-GPU parity of the CUDA stage layers against the oracle (oracle/gpt2.py == HF GPT-2 math), through
``oobleck_b200.execution.layer.Layer`` -> C ABI.  Tolerance: north_star's 1e-4 rtol (fp32)."""
import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

if not torch.cuda.is_available():
    pytest.skip("needs CUDA", allow_module_level=True)

from oobleck_b200.execution.layer import HiddenGrad, Layer, StageWorkspace  # noqa: E402
from oobleck_b200.module.model import OobleckModel  # noqa: E402
from oracle import gpt2 as og  # noqa: E402

RTOL = 1e-4


def close(got, want, name, rtol=RTOL):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    scale = want.abs().max().clamp_min(1e-30)
    err = ((got - want).abs().max() / scale).item()
    assert err < rtol, f"{name}: max|err|/max|ref| = {err:.3e}"
    return err


def build(cfg, mb, nbuf=2, nsplit=3, bwd_fp16=False):
    d = og.GPT2Dims(**cfg)
    olayers = og.build_layers(d)
    og.init_layers_(olayers)
    # make LayerNorm/bias parameters non-trivial
    g = torch.Generator().manual_seed(7)
    for l in olayers:
        for n, p in l.named_parameters():
            if n.endswith("_b") or n.startswith("ln_"):
                with torch.no_grad():
                    p.add_(torch.randn(p.shape, generator=g) * 0.05)
    model = OobleckModel("gpt2", {"input_ids": None, "attention_mask": None, "labels": None}, None, "test",
                         dict(n_embd=d.n_embd, n_head=d.n_head, n_layer=d.n_layer, n_positions=d.n_positions,
                              vocab_size=d.vocab_size))
    assert len(model.layers) == d.n_layer + 2
    ws = StageWorkspace(mb, d.n_positions, d.n_embd, d.n_head, torch.device("cuda"))
    layers = []
    for i, spec in enumerate(model.layers):
        assert spec.num_params == sum(p.numel() for p in olayers[i].parameters())
        l = Layer(i, spec, None, None, None, microbatch_size=mb, num_pipe_buffers=nbuf, workspace=ws, nsplit=nsplit,
                  bwd_fp16=bwd_fp16)
        l.load_flat_(og.flat_params(olayers[i]))
        layers.append(l)
    return d, olayers, layers


@pytest.mark.parametrize("bwd_fp16", [False, True])
@pytest.mark.parametrize("cfg,mb", [
    (dict(n_embd=128, n_head=2, n_layer=2, n_positions=64, vocab_size=503), 2),
    (dict(n_embd=256, n_head=4, n_layer=3, n_positions=256, vocab_size=1000), 3),
    (dict(n_embd=768, n_head=12, n_layer=2, n_positions=1024, vocab_size=50257), 1),
])
def test_stage_forward_backward_parity(cfg, mb, bwd_fp16):
    d, olayers, layers = build(cfg, mb, bwd_fp16=bwd_fp16)
    total = torch.zeros(1, device="cuda")
    ref_total = 0.0
    n_mb = 2
    for k in range(n_mb):  # two micro-batches: gradients must accumulate
        batch = og.synthetic_batch(mb, d.n_positions, d.vocab_size, index=k)
        x = (batch["input_ids"], batch["attention_mask"], batch["labels"])
        hidden_ref = []
        for ol in olayers:
            x = ol(*x)
            hidden_ref.append(x[0])
        x[0].backward()
        ref_total += x[0].item()

        buf = k % 2
        cx = tuple(t.cuda() for t in (batch["input_ids"], batch["attention_mask"], batch["labels"]))
        for i, l in enumerate(layers):
            cx = l(cx, buffer_id=buf, total_loss=total)
            if i < len(layers) - 1:
                close(cx[0], hidden_ref[i], f"mb{k} hidden after layer {i}")
        close(cx[0], hidden_ref[-1], f"mb{k} loss")
        close(cx[1].view(mb, d.n_positions, -1)[..., :d.vocab_size], x[1], f"mb{k} logits")
        g = None
        for l in reversed(layers):
            g = l.backward(buf, g)
        assert g is None
        layers[0].workspace.join()    # what PipelineExecution.backward_pass does after the last layer
    torch.cuda.synchronize()
    assert abs(total.item() - ref_total) < RTOL * abs(ref_total)
    worst = 0.0
    for i, (l, ol) in enumerate(zip(layers, olayers)):
        worst = max(worst, close(l.flat_grad, og.flat_grads(ol), f"flat grad of layer {i}"))
    print(f"worst grad err {worst:.3e}")


def _stats(got, want):
    got, want = got.detach().double().cuda().flatten(), want.detach().double().cuda().flatten()
    nz = want != 0
    rms = want[nz].pow(2).mean().sqrt().clamp_min(1e-300) if nz.any() else torch.tensor(1e-300, device="cuda").double()
    return got, want, rms


def elementwise_report(got, want, name):
    """Fraction of elements violating |got - want| <= rtol |want| + atol for rtol = 1e-4 and a few absolute floors,
    the floor expressed in units of rms(want) over the non-zero reference entries."""
    got, want, rms = _stats(got, want)
    err = (got - want).abs()
    out = {f: float((err > 1e-4 * want.abs() + f * rms).double().mean()) for f in (1e-6, 1e-5, 1e-4)}
    print(f"  {name:30s} max|err|/max|ref| {float(err.max() / want.abs().max()):.2e}  rms(err)/rms {float(err.pow(2).mean().sqrt() / rms):.2e}"
          f"  violations at atol (1e-6, 1e-5, 1e-4) x rms: {out[1e-6]:.2e} {out[1e-5]:.2e} {out[1e-4]:.2e}", flush=True)
    return out


# Elementwise bar (north_star "1e-4 rtol fp32"): |got - ref| <= RTOL * |ref| + ATOL_RMS * rms(ref) for EVERY element,
# ref = the oracle evaluated in float64, rms over the non-zero reference entries (embedding gradients are mostly exact
# zeros).  Some absolute floor is needed by ANY fp32 implementation: an entry that is the sum of K products of typical
# size s carries ~sqrt(K) 2^-24 s of rounding noise however small the entry itself comes out.  At the GPT-2-XL dims the
# test prints the share of violating elements of the engine next to that of torch's own fp32 CUDA path (the reference's
# arithmetic: SGEMM, eager softmax) at the same bar.
ATOL_RMS = 1e-4


def allclose_elementwise(got, want, name, atol_rms=ATOL_RMS):
    got, want, rms = _stats(got, want)
    bad = (got - want).abs() > RTOL * want.abs() + atol_rms * rms
    assert not bool(bad.any()), f"{name}: {int(bad.sum())} of {bad.numel()} elements outside rtol {RTOL} + {atol_rms} rms"


@pytest.mark.parametrize("bwd_fp16", [False, True])
def test_stage_parity_at_benchmark_dims(bwd_fp16):
    """The configuration bench.py times (GPT-2-XL: E=1600, H=25, T=1024, micro-batch 2, loss scale 16384 in fp16-pair
    mode), at reduced depth: embedding + 2 blocks + head, two micro-batches.  Reference = oracle/gpt2.py evaluated in
    float64 (on the GPU, for speed); the same oracle in float32 on the GPU -- what the reference itself computes -- is
    reported next to it."""
    import copy
    cfg = dict(n_embd=1600, n_head=25, n_layer=2, n_positions=1024, vocab_size=50257)
    mb = 2
    d, olayers, layers = build(cfg, mb, bwd_fp16=bwd_fp16)
    o32 = [copy.deepcopy(l).cuda() for l in olayers]
    o64 = [copy.deepcopy(l).double().cuda() for l in olayers]
    del olayers
    total = torch.zeros(1, device="cuda")
    ref_total = 0.0
    for k in range(2):
        batch = og.synthetic_batch(mb, d.n_positions, d.vocab_size, index=k)
        x64 = x32 = cx = tuple(t.cuda() for t in (batch["input_ids"], batch["attention_mask"], batch["labels"]))
        h64 = []
        for l32, l64 in zip(o32, o64):
            x32 = l32(*x32)
            x64 = l64(*x64)
            h64.append(x64[0].detach())
        x32[0].backward()
        x64[0].backward()
        ref_total += x64[0].item()
        del x32, x64
        for i, l in enumerate(layers):
            cx = l(cx, buffer_id=k, total_loss=total)
            if i < len(layers) - 1:
                close(cx[0], h64[i], f"mb{k} hidden after layer {i}", rtol=1e-5)
                allclose_elementwise(cx[0], h64[i], f"mb{k} hidden after layer {i}")
        assert abs(cx[0].item() - h64[-1].item()) < 1e-5 * abs(h64[-1].item())
        g = None
        for l in reversed(layers):
            g = l.backward(k, g)
        layers[0].workspace.join()
    torch.cuda.synchronize()
    assert abs(total.item() - ref_total) < 1e-5 * abs(ref_total)
    print(f"\nbwd_fp16={bwd_fp16}: flat gradients vs the float64 oracle -- CUDA engine | torch float32 on the same GPU")
    for i, (l, l32, l64) in enumerate(zip(layers, o32, o64)):
        want = og.flat_grads(l64)
        elementwise_report(l.flat_grad, want, f"layer {i} ({l.spec.kind}) engine")
        elementwise_report(og.flat_grads(l32), want, f"layer {i} ({l.spec.kind}) torch f32")
    for i, (l, l64) in enumerate(zip(layers, o64)):
        want = og.flat_grads(l64)
        close(l.flat_grad, want, f"flat grad of layer {i}", rtol=1e-5)
        allclose_elementwise(l.flat_grad, want, f"flat grad of layer {i}")


@pytest.mark.parametrize("shift", [-10, 0, 10])
def test_block_backward_loss_scale_stress(shift):
    """fp16-pair backward: the incoming gradient is 2^shift times its usual loss-scaled magnitude (gradients far
    smaller / larger than the scale was chosen for).  dx and every parameter gradient must keep the parity bar."""
    cfg = dict(n_embd=256, n_head=4, n_layer=1, n_positions=256, vocab_size=300)
    mb = 2
    d, olayers, layers = build(cfg, mb, bwd_fp16=True)
    blk, oblk = layers[1], olayers[1]
    g = torch.Generator().manual_seed(3)
    x = torch.randn(mb, d.n_positions, d.n_embd, generator=g)
    labels = torch.zeros(mb, d.n_positions, dtype=torch.int64)
    dy = torch.randn(mb, d.n_positions, d.n_embd, generator=g) * 1e-4     # a typical d(loss)/d(hidden) magnitude
    x64 = x.double().requires_grad_(True)
    o6 = __import__("copy").deepcopy(oblk).double()
    y64 = o6(x64, labels)[0]
    y64.backward(dy.double())
    blk((x.cuda().contiguous(), labels.cuda()), buffer_id=0)
    f = blk.loss_scale * 2.0 ** shift
    out = blk.backward(0, HiddenGrad((dy * f).cuda().contiguous()))
    blk.workspace.join()
    torch.cuda.synchronize()
    close(out.grad.view_as(x).cpu() / f, x64.grad, "dx", rtol=1e-5)
    # parameter gradients are unscaled by 1/loss_scale inside the kernels: they come out 2^shift times the true ones
    close(blk.flat_grad.cpu() / 2.0 ** shift, og.flat_grads(o6), "flat grad", rtol=1e-5)
    allclose_elementwise(blk.flat_grad.cpu() / 2.0 ** shift, og.flat_grads(o6), "flat grad")


def test_stage_split_levels_accuracy():
    """nsplit=3 must be the most accurate; nsplit=1 is plain bf16 and must NOT meet the parity tolerance."""
    cfg = dict(n_embd=256, n_head=4, n_layer=2, n_positions=128, vocab_size=777)
    errs = {}
    for ns in (3, 2, 1):
        d, olayers, layers = build(cfg, 2, nsplit=ns)
        batch = og.synthetic_batch(2, d.n_positions, d.vocab_size)
        x = (batch["input_ids"], batch["attention_mask"], batch["labels"])
        for ol in olayers:
            x = ol(*x)
        cx = tuple(t.cuda() for t in (batch["input_ids"], batch["attention_mask"], batch["labels"]))
        for l in layers[:-1]:
            cx = l(cx, buffer_id=0)
        ref_h = None
        x2 = (batch["input_ids"], batch["attention_mask"], batch["labels"])
        for ol in olayers[:-1]:
            x2 = ol(*x2)
        errs[ns] = ((cx[0].cpu().double() - x2[0].double()).abs().max() / x2[0].double().abs().max()).item()
    print(errs)
    assert errs[3] < 1e-5 and errs[3] <= errs[2] <= errs[1]
    assert errs[1] > 1e-4


def test_adamw_layer_step_matches_oracle():
    import ctypes as C

    from oobleck_b200 import lib as L
    from oracle import optim as oo
    cfg = dict(n_embd=128, n_head=2, n_layer=1, n_positions=64, vocab_size=300)
    d, olayers, layers = build(cfg, 1)
    l = layers[1]
    p = l.flat_param.clone().cpu()
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    for step in range(1, 4):
        g = torch.randn(l.numel)
        l.flat_grad.copy_(g)
        lr = 1e-3 * step
        L.call("oob_adamw_step", C.c_void_p(l.flat_param.data_ptr()), C.c_void_p(l.flat_grad.data_ptr()),
               C.c_void_p(l.exp_avg.data_ptr()), C.c_void_p(l.exp_avg_sq.data_ptr()), C.c_void_p(l.planes.data_ptr()),
               l.plane_stride, l.nplanes, l.numel, lr, 0.9, 0.999, 1e-8, 0.01, step,
               C.c_void_p(torch.cuda.current_stream().cuda_stream))
        oo.adamw_step_(p, g, m, v, step, lr)
        close(l.flat_param, p, f"param after step {step}", rtol=1e-6)
    if l.nplanes != L.PLANES_FP16_PAIR:
        close(l.planes[:3, :l.numel].float().sum(0), p, "bf16 planes track the parameters", rtol=1e-6)
    if l.nplanes in (L.PLANES_BF16X3_FP16_PAIR, L.PLANES_FP16_PAIR):   # pair at planes 3, 4 / at 0, 1 of a pair-only one
        o = 3 if l.nplanes == L.PLANES_BF16X3_FP16_PAIR else 0
        h = l.planes[o:o + 2, :l.numel].view(torch.float16).float()
        close(h[0] + h[1] / 2048.0, p, "fp16 pair tracks the parameters", rtol=1e-6)


def test_side_stream_wgrad_is_bit_identical():
    """Weight gradients computed on the side stream (overlapped with the dgrad chain) must equal, bit for bit, the
    ones computed with every kernel on the caller's stream."""
    import ctypes as C
    from oobleck_b200 import lib as L
    cfg = dict(n_embd=256, n_head=4, n_layer=3, n_positions=256, vocab_size=1000)
    grads = {}
    for on in (1, 0):
        L.call("oob_side_stream_enable", on)
        try:
            d, olayers, layers = build(cfg, 2)
            for k in range(3):
                batch = og.synthetic_batch(2, d.n_positions, d.vocab_size, seed=k)
                cx = tuple(t.cuda() for t in (batch["input_ids"], batch["attention_mask"], batch["labels"]))
                for l in layers:
                    cx = l(cx, buffer_id=k % 2)
                g = None
                for l in reversed(layers):
                    g = l.backward(k % 2, g)
                layers[0].workspace.join()
            torch.cuda.synchronize()
            grads[on] = [l.flat_grad.clone() for l in layers]
        finally:
            L.call("oob_side_stream_enable", 1)
    # layer 0 (embedding) scatters with float atomics -- run-to-run order differs with or without the side stream
    for i, (a, b) in enumerate(zip(grads[1], grads[0])):
        if i == 0:
            assert torch.allclose(a, b, rtol=1e-5, atol=1e-8)
        else:
            assert torch.equal(a, b), f"layer {i}"
