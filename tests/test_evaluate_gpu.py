"""``OobleckEngine.evaluate`` on one GPU at the benchmark's width (GPT-2-XL: E = 1600, 25 heads, T = 1024,
V = 50257) and reduced depth (embedding + 2 blocks + head): the loss against the float64 oracle, the memory an
evaluation at micro-batch 8 needs, and training steps with an evaluation in between."""
import math

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

if not torch.cuda.is_available():
    pytest.skip("needs CUDA", allow_module_level=True)

from oobleck_b200.execution.dataloader import SyntheticTokenDataset  # noqa: E402
from oobleck_b200.execution.engine import JobArguments, ModelArguments, OobleckArguments, OobleckEngine  # noqa: E402
from oracle import gpt2 as og  # noqa: E402

MARGS = dict(n_embd=1600, n_head=25, num_hidden_layers=2, n_positions=1024, vocab_size=50257)
TRAIN_MB, EVAL_MB, N_EVAL = 2, 8, 2


def make_engine():
    torch.cuda.set_device(0)
    args = OobleckArguments(job=JobArguments(microbatch_size=TRAIN_MB, global_microbatch_size=2 * TRAIN_MB, steps=2,
                                             eval_microbatch_size=EVAL_MB),
                            model=ModelArguments(model_name="gpt2", model_tag="xl-2", model_args=dict(MARGS)))
    ds = SyntheticTokenDataset(num_samples=32, seq_len=1024, vocab_size=50257)
    # every token id at most once in the whole set: the embedding backward accumulates repeated ids with atomics, the
    # one place where a training step is not bit-reproducible by itself
    g = torch.Generator().manual_seed(1)
    ds.input_ids = torch.randperm(50257, generator=g)[:32 * 1024].view(32, 1024).contiguous().pin_memory()
    eng = OobleckEngine(0, 1, 1, None, args, dataset=ds)
    eng.initialize_distributed()
    eng.instantiate_pipelines(2)
    return eng, ds


def oracle_loss(eng, ds):
    """float64 oracle (on the GPU) over the same validation micro-batches: mean of the micro-batch mean losses."""
    d = og.GPT2Dims(n_embd=1600, n_head=25, n_layer=2, n_positions=1024, vocab_size=50257)
    olayers = og.build_layers(d)
    for ol, l in zip(olayers, eng._pipeline.execution._layers):
        og.load_flat_(ol, l.flat_param.cpu())
    olayers = [ol.double().cuda() for ol in olayers]
    losses = []
    with torch.no_grad():
        for k in range(N_EVAL):
            ids = ds.input_ids[k * EVAL_MB:(k + 1) * EVAL_MB].cuda()
            x = (ids, torch.ones_like(ids), ids)
            for ol in olayers:
                x = ol(*x)
            losses.append(float(x[0]))
    del olayers
    torch.cuda.empty_cache()
    return sum(losses) / len(losses)


def test_evaluate_matches_fp64_oracle_and_fits_in_one_training_microbatch():
    eng, ds = make_engine()
    layers = eng._pipeline.execution._layers
    # what ONE training micro-batch keeps alive through its backward: every layer's context and output of one slot
    train_ctx = sum(t.numel() * t.element_size() for l in layers for t in l.ctx_tensors[0].values())
    train_ctx += sum(l.out[0].numel() * l.out[0].element_size() for l in layers)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    got = eng.evaluate(N_EVAL)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    print(f"evaluate at micro-batch {EVAL_MB}: peak {peak / 2**20:.0f} MiB; one training micro-batch ({TRAIN_MB}) "
          f"keeps {train_ctx / 2**20:.0f} MiB of contexts")
    assert peak < train_ctx
    assert got["microbatches"] == N_EVAL and got["tokens"] == N_EVAL * EVAL_MB * 1023
    assert got["perplexity"] == math.exp(got["loss"])
    want = oracle_loss(eng, ds)
    print(f"evaluate loss {got['loss']:.9f}, float64 oracle {want:.9f}")
    assert abs(got["loss"] - want) <= 1e-5 * abs(want)
    assert eng.evaluate(N_EVAL) == got        # the same bits again: deterministic, starts at the split's beginning


def _training_state(eng) -> dict:
    torch.cuda.synchronize()
    pipe = eng._pipeline
    ex = pipe.execution
    return {
        "params": [l.flat_param.detach().clone() for l in ex._layers],
        "grads": [l.flat_grad.detach().clone() for l in ex._layers],
        "m": [l.exp_avg.detach().clone() for l in ex._layers],
        "v": [l.exp_avg_sq.detach().clone() for l in ex._layers],
        "planes": [l.planes.clone() for l in ex._layers if l.planes is not None],
        "total_loss": float(ex.total_loss) if ex.total_loss is not None else None,
        "step": pipe._global_step,
        "lr": ex._optimizer.param_groups[0]["lr"],
        "opt_step": [l.opt_step for l in ex._layers],
    }


def _assert_same(a: dict, b: dict):
    for k, x in a.items():
        if isinstance(x, list) and x and isinstance(x[0], torch.Tensor):
            bad = [i for i, (p, q) in enumerate(zip(x, b[k])) if not torch.equal(p.view(torch.int16), q.view(torch.int16))]
            assert not bad, f"{k} differs in layers {bad}"
        else:
            assert x == b[k], (k, x, b[k])


def test_evaluate_leaves_training_state_untouched():
    eng, _ = make_engine()
    eng._train_step()
    before = _training_state(eng)
    eng.evaluate(N_EVAL)
    _assert_same(before, _training_state(eng))


def _train(steps: int, evaluate_between: bool) -> dict:
    eng, _ = make_engine()
    losses = []
    for i in range(steps):
        if evaluate_between and i > 0:
            eng.evaluate(N_EVAL)
        eng._train_step()
        losses.append(float(eng._pipeline.execution.total_loss))
    out = _training_state(eng)
    out["losses"] = losses
    del eng
    torch.cuda.empty_cache()
    return out


def test_training_with_evaluate_between_steps_is_bit_identical():
    a = _train(3, False)
    b = _train(3, True)
    assert a["step"] == 3
    _assert_same(a, b)
