"""``OobleckEngine.evaluate`` on CPU + gloo with the oracle as stage compute: the forward-only program simulated over a
grid of (micro-batches, stages), then real multi-process runs on 1, 2 and 4 stages and on 2 replicas, against a
single-process oracle loss.  Evaluation micro-batches larger than the training micro-batch -- also a size that is not
a multiple of it -- cross the stage boundaries in slices of one training micro-batch."""
import math
import os
import sys

import pytest
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oobleck_b200.execution.schedule import (ForwardPass, LoadMicroBatch, OobleckEvalSchedule,  # noqa: E402
                                             RecvActivation, SendActivation)

MARGS = dict(n_embd=64, n_head=1, num_hidden_layers=2, n_positions=32, vocab_size=211)
NUM_SAMPLES = 128   # the training data of test_pipeline_gloo.reference_run


# ---- simulation ------------------------------------------------------------------------------------------------------
def simulate(micro_batches: int, stages: int):
    """Run every stage's program with blocking rendezvous transfers: a SendActivation completes only together with the
    matching RecvActivation of the next stage.  Each stage has one output buffer (written by ForwardPass, read by the
    send) and one input buffer (written by a load or a receive, read by ForwardPass).  Returns the forwarded micro-batch
    ids per stage; raises on deadlock or on a buffer written while its previous contents are still unread."""
    progs = [[c for step in OobleckEvalSchedule(micro_batches, stages, s) for c in step] for s in range(stages)]
    pc = [0] * stages
    loaded = [0] * stages                 # next micro-batch id a LoadMicroBatch reads
    inp = [None] * stages                 # micro-batch id held in the input buffer (None: consumed)
    out = [None] * stages                 # micro-batch id held in the output buffer, not yet sent
    forwarded = [[] for _ in range(stages)]
    while any(pc[s] < len(progs[s]) for s in range(stages)):
        progressed = False
        for s in range(stages):
            if pc[s] >= len(progs[s]):
                continue
            cmd = progs[s][pc[s]]
            if isinstance(cmd, LoadMicroBatch):
                assert inp[s] is None, f"stage {s}: input buffer overwritten before its forward"
                inp[s] = loaded[s]
                loaded[s] += 1
            elif isinstance(cmd, ForwardPass):
                assert inp[s] is not None, f"stage {s}: forward without input"
                assert out[s] is None, f"stage {s}: output buffer overwritten before it was sent"
                forwarded[s].append(inp[s])
                # the last stage's output is the loss, consumed by the forward itself
                out[s], inp[s] = (inp[s] if s < stages - 1 else None), None
            elif isinstance(cmd, SendActivation):
                peer = progs[s + 1][pc[s + 1]] if pc[s + 1] < len(progs[s + 1]) else None
                if not isinstance(peer, RecvActivation):
                    continue                   # blocked until the next stage posts its receive
                assert inp[s + 1] is None, f"stage {s + 1}: input buffer overwritten before its forward"
                inp[s + 1], out[s] = out[s], None
                pc[s + 1] += 1
            elif isinstance(cmd, RecvActivation):
                continue                       # completes together with the previous stage's send
            pc[s] += 1
            progressed = True
        if not progressed:
            raise RuntimeError(f"deadlock at {pc} for {micro_batches} micro-batches on {stages} stages")
    return forwarded


@pytest.mark.parametrize("stages", [1, 2, 3, 4, 5, 8])
@pytest.mark.parametrize("micro_batches", [0, 1, 2, 3, 7, 16])
def test_eval_schedule_simulation(micro_batches, stages):
    forwarded = simulate(micro_batches, stages)
    for s in range(stages):
        assert forwarded[s] == list(range(micro_batches)), (s, forwarded[s])


def test_eval_schedule_program_shape():
    assert OobleckEvalSchedule(3, 1, 0).program == [[LoadMicroBatch(0), ForwardPass(0)]] * 3
    assert OobleckEvalSchedule(2, 3, 0).program == [[LoadMicroBatch(0), ForwardPass(0), SendActivation(0)]] * 2
    assert OobleckEvalSchedule(2, 3, 1).program == [[RecvActivation(0), ForwardPass(0), SendActivation(0)]] * 2
    assert OobleckEvalSchedule(2, 3, 2).program == [[RecvActivation(0), ForwardPass(0)]] * 2
    assert OobleckEvalSchedule(5, 4, 2).num_pipe_buffers() == 1


# ---- multi-process runs ------------------------------------------------------------------------------------------------
def make_engine(rank, world, mb, eval_mb, M, templates=None):
    from oracle_eval_layer import EvalOracleLayer
    from oobleck_b200.execution.dataloader import SyntheticTokenDataset
    from oobleck_b200.execution.engine import JobArguments, ModelArguments, OobleckArguments, OobleckEngine
    args = OobleckArguments(job=JobArguments(microbatch_size=mb, global_microbatch_size=mb * M, steps=2,
                                             eval_microbatch_size=eval_mb),
                            model=ModelArguments(model_name="gpt2", model_tag="t", model_args=dict(MARGS)))
    ds = SyntheticTokenDataset(num_samples=NUM_SAMPLES, seq_len=32, vocab_size=211, pin_memory=False)
    eng = OobleckEngine(rank, world, 1, None, args, dataset=ds, layer_cls=EvalOracleLayer,
                        templates=templates)
    eng.initialize_distributed("gloo")
    return eng


def reference_eval(eval_mb, n):
    """Single process: the oracle model at its initial weights over the first n validation micro-batches in order."""
    from oobleck_b200.execution.dataloader import SyntheticTokenDataset
    from oobleck_b200.module.model import OobleckModel
    from oracle import gpt2 as og
    model = OobleckModel("gpt2", {"input_ids": None, "attention_mask": None, "labels": None}, None, "t", dict(MARGS))
    d = og.GPT2Dims(n_embd=64, n_head=1, n_layer=2, n_positions=32, vocab_size=211)
    layers = og.build_layers(d)
    for l, spec in zip(layers, model.layers):
        og.load_flat_(l, spec.init_flat())
    ds = SyntheticTokenDataset(num_samples=NUM_SAMPLES, seq_len=32, vocab_size=211, pin_memory=False)
    losses = []
    with torch.no_grad():
        for k in range(n):
            ids = ds.input_ids[k * eval_mb:(k + 1) * eval_mb]
            x = (ids, torch.ones_like(ids), ids)
            for l in layers:
                x = l(*x)
            losses.append(float(x[0]))
    return sum(losses) / n, n * eval_mb * 31


def worker_eval(rank, world, port, mb, eval_mb, n_eval, replicas, train_between, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.set_num_threads(2)
    try:
        from oobleck_b200.planning.pipeline_template import even_template
        M = 4
        templates = [even_template(4, world // replicas)] if replicas > 1 else None
        eng = make_engine(rank, world, mb, eval_mb, M, templates)
        eng.instantiate_pipelines(M)
        pipe = eng._pipeline
        assert len(eng._reconfiguration._pipelines) == replicas
        first = eng.evaluate(n_eval)
        again = eng.evaluate(n_eval)            # every call starts at the beginning of the validation split
        flats = None
        if train_between:
            eng._train_step()
            eng.evaluate(n_eval)
            eng._train_step()
            assert pipe._global_step == 2
            flats = {l.layer_id: l.flat_param.detach().clone().numpy() for l in pipe.execution._layers}
        q.put((rank, (first, again, flats), None, None))
        if dist.is_initialized():
            dist.barrier()
    except Exception:  # noqa: BLE001
        import traceback
        q.put((rank, None, None, traceback.format_exc()))
        raise


def run(world, *a):
    from test_pipeline_gloo import run_spawn
    res = run_spawn(worker_eval, world, *a)
    return [r[1] for r in res]


@pytest.mark.timeout(300)
@pytest.mark.parametrize("world,replicas,mb,eval_mb,n_eval", [
    (1, 1, 2, 3, 5),      # single stage
    (2, 1, 2, 4, 3),      # eval micro-batch = 2 training micro-batches per transfer
    (2, 1, 2, 5, 4),      # not a multiple: slices of 2, 2, 1 sequences
    (4, 1, 1, 3, 6),      # four stages
    (2, 2, 2, 3, 5),      # two single-stage replicas: 3 + 2 micro-batches
])
def test_evaluate_matches_single_process_oracle(world, replicas, mb, eval_mb, n_eval):
    outs = run(world, mb, eval_mb, n_eval, replicas, False)
    want, tokens = reference_eval(eval_mb, n_eval)
    for first, again, _ in outs:                 # every rank returns the same dict
        assert first == outs[0][0] and again == first
        assert first["microbatches"] == n_eval and first["tokens"] == tokens
        assert abs(first["loss"] - want) <= 1e-5 * abs(want), (first["loss"], want)
        assert first["perplexity"] == math.exp(first["loss"])


@pytest.mark.timeout(300)
def test_evaluate_between_steps_leaves_training_unchanged():
    """Two training steps with evaluations before and between them end at the parameters of two plain steps."""
    from test_pipeline_gloo import reference_run
    outs = run(2, 1, 3, 2, 1, True)
    flats, _, _ = reference_run(4, 1, 2)
    seen = {}
    for _, _, f in outs:
        seen.update(f)
    assert sorted(seen) == [0, 1, 2, 3]
    for lid, f in seen.items():
        torch.testing.assert_close(torch.from_numpy(f), flats[lid], rtol=1e-5, atol=1e-7)


def worker_too_many(rank, world, port, q):
    """Asking for more micro-batches than the validation split holds raises on EVERY rank before any transfer, and the
    pipeline stays usable."""
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.set_num_threads(2)
    try:
        eng = make_engine(rank, world, 2, 4, 4)
        eng.instantiate_pipelines(4)
        available = NUM_SAMPLES // 4
        for n in (available + 1, 0):
            try:
                eng.evaluate(n)
            except ValueError as e:
                assert "validation split holds" in str(e)
            else:
                raise AssertionError(f"evaluate({n}) did not raise")
        got = eng.evaluate(available)
        q.put((rank, got, None, None))
        if dist.is_initialized():
            dist.barrier()
    except Exception:  # noqa: BLE001
        import traceback
        q.put((rank, None, None, traceback.format_exc()))
        raise


@pytest.mark.timeout(300)
def test_evaluate_rejects_more_microbatches_than_the_split_holds():
    from test_pipeline_gloo import run_spawn
    outs = [r[1] for r in run_spawn(worker_too_many, 2)]
    assert outs[0] == outs[1] and outs[0]["microbatches"] == NUM_SAMPLES // 4
