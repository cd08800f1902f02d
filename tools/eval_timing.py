"""Evaluation throughput and the cost of the LM head with and without logits, on one GPU.

    python tools/eval_timing.py [--layers 48] [--eval-mb 8] [--microbatches 4] [--reps 5]

1. The head at GPT-2-XL width (E = 1600, V = 50257, T = 1024) for M = 2048 and 8192 rows: the training head
   ``oob_head_forward`` (fp32 logits [M, 50304], dlogits planes, cross entropy) against the forward-only
   ``oob_head_eval`` (row log-sum-exp partials, no logits): milliseconds per call and the bytes of the buffers each needs.
2. ``OobleckEngine.evaluate`` on GPT-2-XL (``--layers`` blocks): validation tokens per second at ``--eval-mb``.

Every figure is printed with the card's name and power limit, which are part of the number.  Times are CUDA-event
medians over ``--reps`` calls after one warm-up call."""
from __future__ import annotations

import argparse
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def card() -> str:
    name = torch.cuda.get_device_name()
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                                str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = limit.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return f"{name}, power limit {power}"


def median_ms(fn, reps: int) -> float:
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times)


def head_timing(reps: int, where: str) -> None:
    from oobleck_b200.execution.layer import EvalWorkspace, Layer
    from oobleck_b200.module.model import OobleckModel
    E, V, T = 1600, 50257, 1024
    model = OobleckModel("gpt2", {"input_ids": None, "attention_mask": None, "labels": None}, None, "xl",
                         dict(n_embd=E, n_head=25, n_layer=1, n_positions=T, vocab_size=V))
    spec = model.layers[-1]
    for M in (2048, 8192):
        B = M // T
        head = Layer(len(model.layers) - 1, spec, None, None, None, microbatch_size=B, num_pipe_buffers=1)
        x = torch.randn(B, T, E, device="cuda")
        labels = torch.randint(0, V, (B, T), device="cuda")
        ws = EvalWorkspace(B, T, E, 25, V, torch.device("cuda"))
        t_fwd = median_ms(lambda: head.forward((x, labels), 0), reps)
        t_eval = median_ms(lambda: head.evaluate((x, labels), ws), reps)
        fwd_bytes = sum(t.numel() * t.element_size() for t in head.ctx_tensors[0].values())
        eval_bytes = sum(t.numel() * t.element_size() for b in ws._head.values() for t in b.values())
        print(f"head M={M}: oob_head_forward {t_fwd:.3f} ms ({fwd_bytes / 2**20:.0f} MiB of buffers), "
              f"oob_head_eval {t_eval:.3f} ms ({eval_bytes / 2**20:.0f} MiB)  [{where}]", flush=True)
        del head, ws
        torch.cuda.empty_cache()


def engine_timing(layers: int, eval_mb: int, microbatches: int, reps: int, where: str) -> None:
    from oobleck_b200.execution.dataloader import SyntheticTokenDataset
    from oobleck_b200.execution.engine import JobArguments, ModelArguments, OobleckArguments, OobleckEngine
    margs = dict(n_embd=1600, n_head=25, num_hidden_layers=layers, n_positions=1024, vocab_size=50257)
    args = OobleckArguments(job=JobArguments(microbatch_size=2, global_microbatch_size=2, steps=1,
                                             eval_microbatch_size=eval_mb),
                            model=ModelArguments(model_name="gpt2", model_tag="xl", model_args=margs))
    ds = SyntheticTokenDataset(num_samples=eval_mb * microbatches, seq_len=1024, vocab_size=50257)
    eng = OobleckEngine(0, 1, 1, None, args, dataset=ds)
    eng.initialize_distributed()
    eng.instantiate_pipelines(1)
    eng.evaluate(microbatches)          # warm-up: allocates the evaluation workspace
    torch.cuda.synchronize()
    secs = []
    for _ in range(reps):
        t0 = time.perf_counter()
        r = eng.evaluate(microbatches)  # returns host floats: the device has finished
        secs.append(time.perf_counter() - t0)
    s = statistics.median(secs)
    tokens = eval_mb * microbatches * 1024
    print(f"evaluate GPT-2-XL ({layers} blocks) eval mb {eval_mb} x {microbatches}: {tokens / s:,.0f} tokens/s "
          f"({s * 1e3:.1f} ms per call, loss {r['loss']:.4f}, peak {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB "
          f"allocated)  [{where}]", flush=True)


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--layers", type=int, default=48)
    ap.add_argument("--eval-mb", type=int, default=8)
    ap.add_argument("--microbatches", type=int, default=4)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--skip-engine", action="store_true")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    where = card()
    head_timing(a.reps, where)
    if not a.skip_engine:
        engine_timing(a.layers, a.eval_mb, a.microbatches, a.reps, where)


if __name__ == "__main__":
    main()
