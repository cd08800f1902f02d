"""Inter-stage wire protocol, interoperability with the reference itself (pipeline.py:247-427).

Two gloo processes form a stage boundary; on one side sits this package's ``PipelineCommunication`` + ``DistTransport``,
on the other the REFERENCE's ``PipelineCommunication`` -- replayed from tests/golden/wire_reference.json: every blocking
``send`` / ``recv`` the reference's unmodified class issued in that role (its ``_send`` / ``_recv``, pipeline.py:270-286),
in order, with dtype, shape and contents.  The replay sends the reference's own bytes and checks that what this package
sends is, bit for bit, what the reference received.  In both directions: the one-off meta handshake (count, then ndims /
dtype id / shape / requires_grad per tensor -- ``DTYPE_TO_ID`` on the wire), two micro-batches of activations ``(hidden
fp32 requiring grad, labels int64)``, and the gradient travelling back.

``OOBLECK_REFERENCE=<checkout> python tests/test_wire_protocol_interop.py`` records the file again: it runs the
reference's class (with the stubs of tests/golden/gen_golden.py, ``deepspeed.comm`` delegating to ``torch.distributed``)
against this package's, and checks both sides as this test does.
"""
import json
import os
import sys

import pytest
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from test_pipeline_gloo import run_spawn  # noqa: E402

RECORDED = os.path.join(ROOT, "tests", "golden", "wire_reference.json")


class StagePipeline:
    """What a ``PipelineCommunication`` reads of its pipeline (pipeline.py:266-268, 331, 389, 392, 404, 420)."""

    def __init__(self):
        self.device = torch.device("cpu")
        self.pipe_buffers = {"inputs": [None, None], "labels": [None, None], "outputs": [None, None]}


def microbatch(i):
    g = torch.Generator().manual_seed(100 + i)
    hidden = torch.randn(2, 8, 16, generator=g).requires_grad_(True)
    labels = torch.randint(0, 211, (2, 8), generator=g, dtype=torch.int64)
    return hidden, labels


def gradient(i):
    return torch.randn(2, 8, 16, generator=torch.Generator().manual_seed(200 + i))


def reference_comm(pipeline, prev_rank, next_rank, record):
    """The reference's unmodified class; every ``_send`` / ``_recv`` it issues is appended to ``record``."""
    import gen_golden
    gen_golden.install_stubs()
    import deepspeed.comm as dc
    for name in ("send", "recv", "isend", "irecv", "get_rank", "is_initialized"):
        setattr(dc, name, getattr(dist, name))
    from oobleck.execution.pipeline import PipelineCommunication as ReferenceCommunication
    import oobleck.execution.pipeline as ref_mod
    assert ref_mod.__file__.startswith(os.path.abspath(os.environ["OOBLECK_REFERENCE"]))
    comm = ReferenceCommunication(pipeline, None, prev_rank, next_rank)
    send, recv = comm._send, comm._recv

    def _send(tensor, rank, async_op=False):
        assert not async_op
        record.append({"op": "send", "dtype": str(tensor.dtype), "shape": list(tensor.shape), "data": tensor.tolist()})
        return send(tensor, rank)

    def _recv(tensor, rank, async_op=False):
        assert not async_op
        work = recv(tensor, rank)
        record.append({"op": "recv", "dtype": str(tensor.dtype), "shape": list(tensor.shape), "data": tensor.tolist()})
        return work
    comm._send, comm._recv = _send, _recv
    return comm


def replay(ops, peer):
    """The reference's side of the boundary, from its recorded operations."""
    for op in ops:
        want = torch.tensor(op["data"], dtype=getattr(torch, op["dtype"].split(".")[1])).reshape(op["shape"])
        if op["op"] == "send":
            dist.send(want, peer)
        else:
            got = torch.empty_like(want)
            dist.recv(got, peer)
            assert torch.equal(got, want), (op["dtype"], op["shape"])


def run_sender(comm, pipeline):
    """The earlier stage: sends activations, receives gradients."""
    assert comm.sent_activation_meta is False and comm.grad_recv_buf is None
    for b in (0, 1):
        pipeline.pipe_buffers["outputs"][b] = microbatch(b)
        comm.send_activations(buffer_id=b)
        assert comm.sent_activation_meta is True
    for b in (0, 1):
        comm.recv_gradients(buffer_id=b)
        assert len(comm.grad_recv_buf) == 1                      # one gradient: the labels produce none
        assert torch.equal(comm.grad_recv_buf[0], gradient(b))
        assert comm.grad_recv_buf[0].dtype == torch.float32 and not comm.grad_recv_buf[0].requires_grad


def run_receiver(comm, pipeline):
    """The later stage: receives activations, sends gradients."""
    assert comm.activation_recv_buf is None
    for b in (0, 1):
        comm.recv_activations(buffer_id=b)
        got = pipeline.pipe_buffers["inputs"][b]
        want = microbatch(b)
        assert isinstance(got, tuple) and len(got) == 2
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
        assert got[0].dtype == torch.float32 and got[1].dtype == torch.int64
        assert got[0].requires_grad and not got[1].requires_grad
        assert got[0] is not comm.activation_recv_buf[0]         # cloned out of the reused receive buffer (:386)
    buf_ids = [id(t) for t in comm.activation_recv_buf]
    for b in (0, 1):
        pipeline.pipe_buffers["inputs"][b][0].grad = gradient(b)
        comm.send_gradients(buffer_id=b)
        assert pipeline.pipe_buffers["inputs"][b] is None        # the slot is freed (:404)
    assert [id(t) for t in comm.activation_recv_buf] == buf_ids


def worker(rank, world, port, sender_kind, receiver_kind, q):
    """Kinds: "ours", "reference" (replayed from the recording) or "record" (the reference's class itself)."""
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.set_num_threads(1)
    try:
        dist.init_process_group("gloo")
        pipeline = StagePipeline()
        kind, role = (sender_kind, "sender") if rank == 0 else (receiver_kind, "receiver")
        prev_rank, next_rank = (None, 1) if rank == 0 else (0, None)
        record = []
        if kind == "reference":
            with open(RECORDED) as f:
                replay(json.load(f)[role], 1 - rank)
        else:
            if kind == "ours":
                from oobleck_b200.execution.pipeline import PipelineCommunication
                comm = PipelineCommunication(pipeline, None, prev_rank, next_rank)
            else:
                comm = reference_comm(pipeline, prev_rank, next_rank, record)
            (run_sender if rank == 0 else run_receiver)(comm, pipeline)
        q.put((rank, role, record, None))
        dist.barrier()
    except Exception:  # noqa: BLE001
        import traceback
        q.put((rank, None, None, traceback.format_exc()))
        raise


@pytest.mark.timeout(300)
@pytest.mark.parametrize("sender,receiver", [("reference", "ours"), ("ours", "reference")],
                         ids=["reference-to-this", "this-to-reference"])
def test_stage_boundary_between_the_reference_and_this_package(sender, receiver):
    run_spawn(worker, 2, sender, receiver)


if __name__ == "__main__":
    ref = os.environ.get("OOBLECK_REFERENCE")
    assert ref, "OOBLECK_REFERENCE must name a checkout of the reference project"
    recorded = {}
    for sender, receiver in (("record", "ours"), ("ours", "record")):
        for rank, role, record, _ in run_spawn(worker, 2, sender, receiver):
            if record:
                recorded[role] = record
    with open(RECORDED, "w") as f:
        json.dump(recorded, f)
