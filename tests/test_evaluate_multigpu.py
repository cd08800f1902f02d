"""``OobleckEngine.evaluate`` on a 2-stage pipeline over the NVLink mailbox transport with the CUDA stage layers
(skipped on a 1-GPU box).  Evaluation micro-batches are larger than the training micro-batch -- a multiple of it and
a size that is not -- so they cross the boundary as several slices, one per mailbox message.  Evaluations run before the
first training step (the link is created by the evaluation, sized for the training tuples), between steps and after;
each is checked against the float64 oracle at the parameters of that moment, and training is checked against the
oracle's own training run."""
import itertools
import os
import sys

import pytest
import torch
import torch.multiprocessing as mp

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]
if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
    pytest.skip("needs 2 GPUs", allow_module_level=True)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from test_multigpu import MARGS, free_port, reference_run  # noqa: E402

M, MB, STEPS, N_EVAL = 6, 2, 2, 3


def worker(rank, world, port, eval_mb, q):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    try:
        import torch.distributed as dist

        from oobleck_b200.execution.dataloader import SyntheticTokenDataset
        from oobleck_b200.execution.engine import JobArguments, ModelArguments, OobleckArguments, OobleckEngine
        from oobleck_b200.execution.p2p import NvlinkRingTransport
        from oobleck_b200.planning.pipeline_template import even_template
        torch.cuda.set_device(rank)
        args = OobleckArguments(job=JobArguments(microbatch_size=MB, global_microbatch_size=MB * M, steps=STEPS,
                                                 eval_microbatch_size=eval_mb),
                                model=ModelArguments(model_name="gpt2", model_tag="t", model_args=dict(MARGS)))
        ds = SyntheticTokenDataset(num_samples=256, seq_len=128, vocab_size=1000)
        eng = OobleckEngine(rank, world, 1, None, args, dataset=ds, templates=[even_template(6, 2)],
                            transport_cls=NvlinkRingTransport)
        eng.initialize_distributed("nccl")
        eng.instantiate_pipelines(M)
        transport = eng._pipeline.communication.transport
        layers = eng._pipeline.execution._layers

        def snapshot():
            return {l.layer_id: l.flat_param.detach().cpu().clone() for l in layers}

        evals, params, totals = [], [], []
        assert not transport.links                  # the first evaluation creates the link
        evals.append(eng.evaluate(N_EVAL))
        params.append(snapshot())
        for _ in range(STEPS):
            eng._train_step()
            tl = eng._pipeline.execution.total_loss
            totals.append(float(tl) if tl is not None else None)
            evals.append(eng.evaluate(N_EVAL))
            params.append(snapshot())
        torch.cuda.synchronize()
        assert not transport.aborted()
        q.put((rank, (evals, params, totals), None))
        dist.barrier()
        dist.destroy_process_group()
    except Exception:  # noqa: BLE001
        import traceback
        q.put((rank, None, traceback.format_exc()))
        raise


def oracle_eval(flats: dict, eval_mb: int) -> float:
    """float64 oracle over the first N_EVAL validation micro-batches: mean of the micro-batch mean losses."""
    from oobleck_b200.execution.dataloader import SyntheticTokenDataset
    from oracle import gpt2 as og
    d = og.GPT2Dims(n_embd=128, n_head=2, n_layer=4, n_positions=128, vocab_size=1000)
    layers = og.build_layers(d)
    for i, l in enumerate(layers):
        og.load_flat_(l, flats[i])
    layers = [l.double() for l in layers]
    ds = SyntheticTokenDataset(num_samples=256, seq_len=128, vocab_size=1000, pin_memory=False)
    losses = []
    with torch.no_grad():
        for k in range(N_EVAL):
            ids = ds.input_ids[k * eval_mb:(k + 1) * eval_mb]
            x = (ids, torch.ones_like(ids), ids)
            for l in layers:
                x = l(*x)
            losses.append(float(x[0]))
    return sum(losses) / N_EVAL


@pytest.mark.parametrize("eval_mb", [4, 5])     # 2 slices of 2 sequences; 2, 2 and 1
def test_evaluate_two_stages_nvlink(eval_mb):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=worker, args=(r, 2, port, eval_mb, q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        results = sorted([q.get(timeout=400) for _ in range(2)], key=lambda r: r[0])
        for p in procs:
            p.join(timeout=60)
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
    for r in results:
        assert r[2] is None, r[2]
    (evals0, params0, _), (evals1, params1, totals) = results[0][1], results[1][1]
    assert evals0 == evals1                      # every rank returns the same dict
    for i, got in enumerate(evals0):
        flats = {**params0[i], **params1[i]}
        assert sorted(flats) == list(range(6))
        want = oracle_eval(flats, eval_mb)
        assert got["microbatches"] == N_EVAL and got["tokens"] == N_EVAL * eval_mb * 127
        assert abs(got["loss"] - want) <= 1e-5 * abs(want), (i, got["loss"], want)
    # training with evaluations in between follows the oracle's training run
    ref_flats, losses = reference_run(M, MB, STEPS, 1)
    final = {**params0[-1], **params1[-1]}
    for lid, f in final.items():
        err = (f - ref_flats[lid]).abs().max() / ref_flats[lid].abs().max()
        assert err < 1e-4, (lid, float(err))
    ref_cum = list(itertools.accumulate(sum(t) for t in losses))
    for got, want in zip(totals, ref_cum):
        assert abs(got - want) < 1e-4 * abs(want)
