"""Pipeline-parallel execution of one Oobleck pipeline on H100s.

Drop-in for oobleck/execution/pipeline.py: same class names, constructor signatures and attributes that the
planner (``HeterogeneousPipelinesExecutionPlan.instantiate``, planning/instantiator.py:135-152), the engine
(execution/engine.py) and the reference's tests touch:

    OobleckPipelineSchedule   1F1B instruction program             (pipeline.py:24-84)     -> .schedule
    PipelineExecution         load / forward / backward / optimizer (pipeline.py:87-245)
    PipelineCommunication     stage <-> stage transfers             (pipeline.py:247-427)
    OobleckPipeline           rank grid, wiring, ``train()``        (pipeline.py:430-623)

What changed underneath:
* stage layers are ``oobleck_b200.execution.layer.Layer`` objects driving hand-written sm_90a kernels, with
  hand-written backward (no autograd graph, no activation recomputation);
* no ``dist.new_group`` per layer / per shard column: membership is plain arithmetic (``RankGroup``), so building or
  re-building a pipeline costs no collective (SURVEY 7 hard part 6);
* activations / gradients move either with the reference's own blocking per-tensor protocol over torch.distributed
  (``DistTransport``: meta handshake then payload; used on CPU/gloo, BASELINE config 1) or as direct NVLink
  peer-memory writes on dedicated streams (``oobleck_b200.execution.p2p.NvlinkRingTransport``).
"""
from __future__ import annotations

import os
import threading
import weakref
from collections.abc import Mapping
from typing import Any

import torch
import torch.distributed as dist

from .dataloader import OobleckDataLoader, OobleckSampler
from .schedule import (BackwardPass, ForwardPass, LoadMicroBatch, OobleckPipelineSchedule, RecvActivation, RecvGrad,
                       SendActivation, SendGrad)
from .utils import DTYPE_TO_ID, ID_TO_DTYPE, zero_grads

__all__ = ["OobleckPipelineSchedule", "PipelineExecution", "PipelineCommunication", "OobleckPipeline", "RankGroup",
           "PipelineAborted"]


class PipelineAborted(RuntimeError):
    """A train step was cut short because a peer was lost (transport abort or communicator abort)."""


def run_interruptible(fn, aborted) -> None:
    """Run a blocking torch.distributed call (gloo) while staying interruptible: the call runs on a helper thread, the
    caller polls ``aborted()`` and leaves with :class:`PipelineAborted` when it fires.  gloo can neither cancel a posted
    operation nor report completion without blocking, so an abandoned call simply stays behind on its daemon thread --
    messages are tagged with the pipeline generation, so an abandoned receive can never match a later message."""
    done = threading.Event()
    err: list[BaseException] = []

    def run():
        try:
            fn()
        except BaseException as e:  # noqa: BLE001
            err.append(e)
        finally:
            done.set()

    threading.Thread(target=run, daemon=True).start()
    while not done.wait(0.002):
        if aborted():
            raise PipelineAborted("transfer abandoned: a peer was lost")
    if err:
        raise err[0]


# every rebuild of the pipelines (initial build = 0, then +1 per reconfiguration) tags its wire traffic differently
_GENERATION = [0]


def bump_generation() -> int:
    _GENERATION[0] += 1
    return _GENERATION[0]


class RankGroup:
    """Membership-only stand-in for a ``torch.distributed.ProcessGroup`` (what ``dist.new_group(list(set(ranks)))``
    returned at pipeline.py:577 / :598).  ``group`` may carry a real communicator when a collective is needed."""

    def __init__(self, ranks: list[int], my_rank: int, group=None):
        self.ranks = list(ranks)
        self.my_rank = my_rank
        self.group = group

    def rank_index(self) -> int:
        return self.ranks.index(self.my_rank) if self.my_rank in self.ranks else -1

    def size(self) -> int:
        return len(self.ranks)


def _my_rank() -> int:
    return dist.get_rank() if dist.is_initialized() else 0


# forward / backward passes of consecutive micro-batches on two CUDA streams (OobleckPipeline.train).  Measured on
# GPT-2-XL, N=1: +2.4 % tokens/s (the step is power-capped: the extra concurrency costs ~100 MHz of SM clock).
# Round 1 applied it to single-stage pipelines only; FB_OVERLAP_PP extends it to the stages of a multi-stage pipeline
# (in the 1F1B steady state every stage alternates one forward and one backward: the same overlap applies).
FB_OVERLAP = os.environ.get("OOB_FB_OVERLAP", "1") == "1"
FB_OVERLAP_PP = os.environ.get("OOB_FB_OVERLAP_PP", "1") == "1"


class PipelineExecution:
    """pipeline.py:87-245."""

    def __init__(self, pipeline: "OobleckPipeline", layers: list, shard_id: int, dataloader: OobleckDataLoader,
                 training_args):
        self._pipeline = weakref.ref(pipeline)
        self._layers = layers
        self._shard_id = shard_id
        self._dataloader = dataloader
        self._data_iterator = iter(self._dataloader)
        self._training_args = training_args
        self._loss: torch.Tensor | None = None       # loss of the micro-batch being processed
        self.total_loss: torch.Tensor | None = None  # running sum over micro-batches (never reset, :196-201)
        self._bwd_seen = 0                           # backward passes so far in this step
        self.grad_ready_hook = None                  # DataParallelEngine.layer_ready when replicas exist

        optimizer_cls, scheduler_cls = pipeline._optimizer_factory()
        self._optimizer = optimizer_cls(
            layers,
            lr=self._training_args.learning_rate,
            betas=(self._training_args.adam_beta1, self._training_args.adam_beta2),
            eps=self._training_args.adam_epsilon,
        )
        num_training_steps = len(self._dataloader)
        # 2nd positional of deepspeed WarmupLR is warmup_min_lr (pipeline.py:125-127) -- kept as is
        # A pipeline rebuilt after a reconfiguration continues the schedule where the job is (``step`` optimizer steps
        # done => the next step reads lr(step - 1), deepspeed's indexing); the reference builds a fresh scheduler
        # (pipeline.py:125-127 inside a new PipelineExecution) and so restarts the warm-up from lr = 0.
        self._lr_scheduler = scheduler_cls(self._optimizer, self._training_args.get_warmup_steps(num_training_steps),
                                           last_batch_iteration=pipeline._global_step - 1)

    @property
    def pipeline(self) -> "OobleckPipeline":
        return self._pipeline()

    def _prepare_input(self, data: torch.Tensor | Any) -> torch.Tensor | Any:  # pipeline.py:134-148
        if isinstance(data, Mapping):
            return type(data)({k: self._prepare_input(v) for k, v in data.items()})
        if isinstance(data, (tuple, list)):
            return type(data)(self._prepare_input(v) for v in data)
        if isinstance(data, torch.Tensor):
            # one async H2D from pinned memory (the reference does clone().detach().to(device), pageable + sync)
            data = data.to(self.pipeline.device, non_blocking=True)
            if data.is_floating_point():
                data.requires_grad = True
            return data
        return data

    def _prepare_inputs(self, inputs: dict[str, torch.Tensor | Any]) -> tuple:  # pipeline.py:150-156
        return tuple(self._prepare_input(t) for _, t in inputs.items())

    def load_microbatch(self, buffer_id: int):
        assert self.pipeline.is_first_stage() or self.pipeline.is_last_stage(), \
            "load_microatch can only be called at either the first stage or the last stage."
        if self.pipeline.is_first_stage():   # the last stage gets its labels through the wire tuple (:163-167)
            batch = next(self._data_iterator)
            self.pipeline.pipe_buffers["inputs"][buffer_id] = self._prepare_inputs(batch)

    def forward_pass(self, buffer_id: int):
        inputs: tuple = self.pipeline.pipe_buffers["inputs"][buffer_id]
        zero_grads(inputs)
        self.pipeline.communication.transport.before_compute()
        if self.pipeline.is_last_stage() and self.total_loss is None:
            self.total_loss = torch.zeros((), dtype=torch.float32, device=self.pipeline.device)
        for layer in self._layers:
            inputs = layer(inputs, buffer_id=buffer_id, total_loss=self.total_loss)
        outputs = inputs
        if self.pipeline.is_last_stage():
            self._loss = outputs[0]          # the layer already did total_loss += loss.detach() on the device
            assert isinstance(self._loss, torch.Tensor)
        else:
            self.pipeline.pipe_buffers["outputs"][buffer_id] = tuple(outputs)

    def backward_pass(self, buffer_id: int):
        from .layer import HiddenGrad
        if self.pipeline.is_last_stage():
            grad = None
        else:
            outputs = self.pipeline.pipe_buffers["outputs"][buffer_id]
            output_tensors = tuple(t for t in outputs if t.requires_grad)
            grad_tensors = self.pipeline.communication.grad_recv_buf
            assert len(output_tensors) == len(grad_tensors)      # pipeline.py:233
            grad = HiddenGrad(grad_tensors[0])
        # the step's LAST micro-batch: a layer's accumulated gradient is final as soon as its backward is enqueued, so
        # the data-parallel engine may start that layer's all-reduce under the backward of the layers before it
        self._bwd_seen = getattr(self, "_bwd_seen", 0) + 1
        hook = self.grad_ready_hook if self._bwd_seen == self.pipeline.train_schedule.micro_batches else None
        for layer in reversed(self._layers):
            grad = layer.backward(buffer_id, grad)
            if hook is not None:
                hook(layer)
        ws = getattr(self._layers[0], "workspace", None)
        if ws is not None and hasattr(ws, "join"):
            ws.join()     # weight-gradient kernels run on a side stream; the ctx slot is recycled after this pass
        if self.pipeline.device.type == "cuda":
            # the stage inputs were allocated under the forward stream (received activations, H2D copies) but this
            # pass reads them on the current stream: tell the allocator, or the block may be handed out again -- to
            # a forward-stream allocation -- while these kernels still read it (send_gradients drops the last reference)
            cur = torch.cuda.current_stream()
            for t in self.pipeline.pipe_buffers["inputs"][buffer_id] or ():
                if isinstance(t, torch.Tensor) and t.is_cuda:
                    t.record_stream(cur)
        if grad is not None:
            # gradient w.r.t. the stage input: parked on the input tensor like autograd would (send_gradients reads
            # ``buffer.grad``, :395-401).  Copied out of the stage's ping-pong buffer because the transfer is async.
            x = self.pipeline.pipe_buffers["inputs"][buffer_id][0]
            x.grad = grad.grad.view_as(x).clone()
        self.pipeline.pipe_buffers["outputs"][buffer_id] = None   # :237
        self._loss = None

    def optimizer_step(self, lr_kwargs=None):
        self._optimizer.step()
        self._lr_scheduler.step(**(lr_kwargs or {}))
        self._optimizer.zero_grad()   # the next step's micro-batches accumulate from zero


class DistTransport:
    """The reference's wire protocol over torch.distributed (pipeline.py:270-427): blocking send/recv of every tuple
    member, preceded once per direction by the int64 meta handshake (count, then ndims / dtype id / shape /
    requires_grad per tensor)."""

    def __init__(self, comm: "PipelineCommunication"):
        self.comm = weakref.ref(comm)
        self._abort = False
        self._tag = _GENERATION[0]

    def _device(self):
        return self.comm().pipeline.device

    # On CPU (gloo) transfers are posted asynchronously and polled, so that a stage waiting for a neighbour that will
    # never answer (lost, or already dropped the step) can be released by ``abort()`` from the listener thread.  NCCL
    # point-to-point (the one-off meta handshake of the NVLink transport) keeps the reference's blocking calls.
    def _interruptible(self) -> bool:
        return self._device().type == "cpu"

    def _send(self, tensor: torch.Tensor, dest_rank: int):
        if not self._interruptible():
            dist.send(tensor.contiguous(), dest_rank, self.comm()._process_group)
            return
        t, pg, tag = tensor.contiguous(), self.comm()._process_group, self._tag
        run_interruptible(lambda: dist.send(t, dest_rank, pg, tag), lambda: self._abort)

    def _recv(self, tensor: torch.Tensor, src_rank: int):
        if not self._interruptible():
            dist.recv(tensor, src_rank, self.comm()._process_group)
            return
        pg, tag = self.comm()._process_group, self._tag
        run_interruptible(lambda: dist.recv(tensor, src_rank, pg, tag), lambda: self._abort)

    def abort(self):
        self._abort = True

    def aborted(self) -> bool:
        return self._abort

    def _long(self, data) -> torch.Tensor:
        return torch.tensor(data, dtype=torch.int64).to(self._device())

    def send_meta(self, buffer: tuple, receiver_rank: int):
        assert isinstance(buffer, tuple), f"Could not send meta type {type(buffer)}."
        self._send(self._long([len(buffer)]), receiver_rank)
        for tensor in buffer:
            assert isinstance(tensor, torch.Tensor)
            self._send(self._long([tensor.dim()]), receiver_rank)
            self._send(self._long([DTYPE_TO_ID[tensor.dtype]]), receiver_rank)
            self._send(self._long(list(tensor.size())), receiver_rank)
            self._send(self._long([1 if tensor.requires_grad else 0]), receiver_rank)

    def recv_meta(self, sender_rank: int) -> tuple:
        count = self._long([0])
        self._recv(count, sender_rank)
        buffers = []
        for _ in range(int(count.item())):
            ndims = self._long([0]); self._recv(ndims, sender_rank)          # noqa: E702
            dtype = self._long([0]); self._recv(dtype, sender_rank)          # noqa: E702
            shape = self._long([1] * int(ndims.item())); self._recv(shape, sender_rank)   # noqa: E702
            req = self._long([0]); self._recv(req, sender_rank)              # noqa: E702
            dt = ID_TO_DTYPE[int(dtype.item())]
            buffers.append(torch.zeros(shape.tolist(), device=self._device(), dtype=dt,
                                       requires_grad=bool(req.item() == 1) and dt.is_floating_point))
        return tuple(buffers)

    def send_tuple(self, tensors, dest_rank: int, kind: str):
        for t in tensors:
            self._send(t, dest_rank)

    def _recv_into(self, buffers, src_rank: int):
        for b in buffers:
            self._recv(b.detach() if b.requires_grad else b, src_rank)

    def recv_activation_tuple(self, recv_buf: tuple, src_rank: int) -> tuple:
        """The receive buffer is reused for every micro-batch and cloned into the pipe buffer (:378-387)."""
        self._recv_into(recv_buf, src_rank)
        recvd = []
        for buffer in recv_buf:
            t = buffer.clone().detach()
            t.requires_grad = buffer.requires_grad
            recvd.append(t)
        return tuple(recvd)

    def recv_gradient_tuple(self, recv_buf: tuple, src_rank: int) -> None:
        self._recv_into(recv_buf, src_rank)

    def before_compute(self) -> None:
        """Called before a forward / backward pass is enqueued; blocking transports have nothing to order."""


class PipelineCommunication:
    """pipeline.py:247-427; attribute names kept (``sent_activation_meta``, ``activation_recv_buf``,
    ``grad_recv_buf``, ``prev_rank``, ``next_rank``)."""

    def __init__(self, pipeline: "OobleckPipeline", process_group, prev_rank: int | None, next_rank: int | None,
                 transport=None):
        self._pipeline = weakref.ref(pipeline)
        self._process_group = process_group
        self.prev_rank = prev_rank
        self.next_rank = next_rank
        self.sent_activation_meta: bool = False
        self.activation_recv_buf: tuple | None = None
        self.grad_recv_buf: tuple | None = None
        self.transport = transport if transport is not None else DistTransport(self)

    @property
    def pipeline(self) -> "OobleckPipeline":
        return self._pipeline()

    def send_activations(self, buffer_id: int):
        outputs: tuple = self.pipeline.pipe_buffers["outputs"][buffer_id]
        assert isinstance(outputs, tuple)
        if not self.sent_activation_meta:
            self.transport.send_meta(outputs, self.next_rank)
            self.sent_activation_meta = True
        self.transport.send_tuple(outputs, self.next_rank, "act")

    def recv_activations(self, buffer_id: int):
        if self.activation_recv_buf is None:
            self.activation_recv_buf = self.transport.recv_meta(self.prev_rank)
        assert isinstance(self.activation_recv_buf, tuple)
        self.pipeline.pipe_buffers["inputs"][buffer_id] = self.transport.recv_activation_tuple(
            self.activation_recv_buf, self.prev_rank)

    def send_gradients(self, buffer_id: int):
        inputs = self.pipeline.pipe_buffers["inputs"][buffer_id]
        assert isinstance(inputs, tuple)
        grads = []
        for buffer in inputs:
            if not buffer.requires_grad:   # tensors that produce no gradient are skipped (:396-399)
                assert buffer.grad is None
                continue
            assert buffer.grad is not None
            grads.append(buffer.grad)
        self.transport.send_tuple(grads, self.prev_rank, "grad")
        self.pipeline.pipe_buffers["inputs"][buffer_id] = None   # :404

    def recv_gradients(self, buffer_id: int):
        outputs = self.pipeline.pipe_buffers["outputs"][buffer_id]
        assert isinstance(outputs, tuple)
        if self.grad_recv_buf is None:     # :407-424
            self.grad_recv_buf = tuple(torch.zeros_like(t, requires_grad=False) for t in outputs if t.requires_grad)
        self.transport.recv_gradient_tuple(self.grad_recv_buf, self.next_rank)


class OobleckPipeline:
    """pipeline.py:430-623."""

    def __init__(self, pipeline_id: int, pipeline_template, ranks: list[int], dataloader: OobleckDataLoader, step: int,
                 training_args, *, layer_cls=None, transport_cls=None, nsplit: int = 3, stage_group_factory=None):
        self._pipeline_id = pipeline_id
        self._template = pipeline_template
        self._ranks = ranks
        self._dataloader = dataloader
        self._global_step = step
        self._training_args = training_args
        self._layer_cls = layer_cls
        self._transport_cls = transport_cls
        self._nsplit = nsplit
        self._stage_group_factory = stage_group_factory    # ranks -> communicator of a multi-GPU stage (tests)
        if layer_cls is not None and hasattr(layer_cls, "device_type"):
            self.device = torch.device(layer_cls.device_type)
        else:
            self.device = torch.device("cuda")           # pipeline.py:446
        # whether this rank trains with this pipeline (:451)
        self.my_pipeline = bool(_my_rank() in ranks)
        # layer index -> list of ranks (:453-456)
        self.rank_grid: dict[int, list[int]] = pipeline_template.get_rank_grid(ranks)
        self.execution: PipelineExecution | None = None
        self.communication: PipelineCommunication | None = None

    # -- training -------------------------------------------------------------------------------------------------
    def train(self):
        instruction_map = {
            LoadMicroBatch: self.execution.load_microbatch,
            ForwardPass: self.execution.forward_pass,
            BackwardPass: self.execution.backward_pass,
            SendActivation: self.communication.send_activations,
            RecvActivation: self.communication.recv_activations,
            SendGrad: self.communication.send_gradients,
            RecvGrad: self.communication.recv_gradients,
        }
        # Forward-family instructions of micro-batch i+1 and backward-family instructions of micro-batch i are
        # independent (weights change only in optimizer_step): with FB_OVERLAP they are enqueued on two CUDA streams,
        # ordered by three kinds of events only -- forward(b) -> backward(b), backward(b) -> next occupant of pipe
        # buffer b, end of step -> optimizer.  The GPU then fills the short last waves / small kernels of one pass
        # with CTAs of the other.  Issue order (the reference's 1F1B program) is unchanged.
        single_stage = self.is_first_stage() and self.is_last_stage()
        overlap = (FB_OVERLAP and self.device.type == "cuda" and torch.cuda.is_available()
                   and (single_stage or FB_OVERLAP_PP))
        prof = getattr(self, "profile", None)   # bench.py: CUDA-event pairs around every forward / backward pass
        if overlap:
            if getattr(self, "_fwd_stream", None) is None:
                self._fwd_stream = torch.cuda.Stream()
            main, fwd = torch.cuda.current_stream(), self._fwd_stream
            fwd.wait_stream(main)                       # previous optimizer step / reconfiguration copies
            fwd_done: dict[int, torch.cuda.Event] = {}
            bwd_done: dict[int, torch.cuda.Event] = {}
        forward_family = (LoadMicroBatch, RecvActivation, ForwardPass, SendActivation)
        self.execution._bwd_seen = 0
        for step_cmds in self.train_schedule:
            for cmd in step_cmds:
                if type(cmd) not in instruction_map:
                    raise RuntimeError(f"{self.__class__.__name__} does not understand instruction {repr(cmd)}")
                timed = prof is not None and type(cmd) in (ForwardPass, BackwardPass)
                if not overlap:
                    if timed:
                        e0 = torch.cuda.Event(enable_timing=True)
                        e0.record()
                    instruction_map[type(cmd)](**cmd.kwargs)
                    if timed:
                        e1 = torch.cuda.Event(enable_timing=True)
                        e1.record()
                        prof.append((type(cmd).__name__, e0, e1))
                    continue
                b = cmd.kwargs.get("buffer_id")
                if type(cmd) in forward_family:
                    with torch.cuda.stream(fwd):
                        if b in bwd_done:               # the previous occupant of this pipe buffer has been consumed
                            fwd.wait_event(bwd_done.pop(b))
                        if timed:
                            e0 = torch.cuda.Event(enable_timing=True)
                            e0.record(fwd)
                        instruction_map[type(cmd)](**cmd.kwargs)
                        if type(cmd) is ForwardPass:
                            fwd_done[b] = torch.cuda.Event(enable_timing=timed)
                            fwd_done[b].record(fwd)
                            if timed:
                                prof.append(("ForwardPass", e0, fwd_done[b]))
                else:
                    if type(cmd) in (BackwardPass, RecvGrad) and b in fwd_done:
                        main.wait_event(fwd_done.pop(b))
                    if timed:
                        e0 = torch.cuda.Event(enable_timing=True)
                        e0.record(main)
                    instruction_map[type(cmd)](**cmd.kwargs)
                    if type(cmd) is BackwardPass:
                        bwd_done[b] = torch.cuda.Event(enable_timing=timed)
                        bwd_done[b].record(main)
                        if timed:
                            prof.append(("BackwardPass", e0, bwd_done[b]))
        if overlap:
            main.wait_stream(fwd)                       # losses, activations still in flight -> optimizer / caller
        for name, pipe_buffers in self.pipe_buffers.items():      # :483-485
            self.pipe_buffers[name] = [None] * len(pipe_buffers)
        self._global_step += 1

    def reset_iterator(self):
        self.execution._data_iterator = iter(self.execution._dataloader)

    # -- construction ---------------------------------------------------------------------------------------------
    def _optimizer_factory(self):
        if self._layer_cls is not None and hasattr(self._layer_cls, "optimizer_factory"):
            return self._layer_cls.optimizer_factory()
        from .optimizer import FusedAdamW, WarmupLR
        return FusedAdamW, WarmupLR

    def initialize_distributed_fsdp(self):
        """Per-layer groups (pipeline.py:565-580).  A layer held by one rank gets membership only; a stage of several
        GPUs shards its layers (layer.py:100-102) and needs a communicator -- ONE per stage, shared by its layers,
        created by its members only (the reference calls ``dist.new_group`` once per layer, on every rank).  Holders
        are listed in rank-grid order, so shard ``j`` of a layer covers the shard columns (``fsdp_index``) where its
        rank stands in the grid row (engine.py:374-384)."""
        me = _my_rank()
        self._per_layer_pgs: dict[int, RankGroup] = {}
        widths = set()
        for layer_id, ranks in self.rank_grid.items():
            holders = list(dict.fromkeys(ranks))
            widths.add(len(holders))
            comm = None
            if len(holders) > 1 and me in holders:
                comm = self._stage_communicator(holders)
            self._per_layer_pgs[layer_id] = RankGroup(holders, me, comm)
        if len(widths) > 1:
            # the reference wires ONE previous and ONE next rank per rank (pipeline.py:602-610): a stage narrower than
            # its neighbour would leave sends without a receiver
            raise NotImplementedError(f"stages of different widths inside one pipeline ({sorted(widths)} GPUs): every "
                                      "stage of a pipeline must own the same number of GPUs")
        self.execution = None

    def _stage_communicator(self, ranks: list[int]):
        if self._stage_group_factory is not None:
            return self._stage_group_factory(ranks)
        from .engine import _COMMUNICATORS, _new_member_group
        key = tuple(sorted(ranks))
        if key not in _COMMUNICATORS:
            _COMMUNICATORS[key] = _new_member_group(key, None)
        return _COMMUNICATORS[key]

    def initialize_distributed_pipeline(self):
        """Per shard column wiring (pipeline.py:582-617): who is my previous / next stage."""
        me = _my_rank()
        self._per_sharded_pp_pgs: dict[int, RankGroup] = {}
        self.communication = None
        first = next(iter(self.rank_grid.values()))
        for shard_id in range(len(first)):
            ranks = [per_layer[shard_id] for per_layer in self.rank_grid.values()]
            unique_ranks = list(set(ranks))     # CPython set order, like the reference (:602-610)
            pg = RankGroup(unique_ranks, me)
            self._per_sharded_pp_pgs[shard_id] = pg
            if me in ranks:
                i = unique_ranks.index(me)
                self.communication = PipelineCommunication(
                    pipeline=self,
                    process_group=None,   # WORLD: send/recv address global ranks, no sub-communicator needed
                    prev_rank=unique_ranks[i - 1] if i > 0 else None,
                    next_rank=unique_ranks[i + 1] if i < len(unique_ranks) - 1 else None,
                )
                if self._transport_cls is not None:
                    self.communication.transport = self._transport_cls(self.communication)
        assert len(self._per_sharded_pp_pgs) == len(first)

    def initialize_execution(self, model, existing_pipeline: "OobleckPipeline | None" = None):
        assert self._per_layer_pgs, "Must call initialize_distributed_fsdp() first"
        my_rank = _my_rank()
        my_layer_index = next(li for li, ranks in self.rank_grid.items() if my_rank in ranks)
        my_stage_index = next(si for si, stage in enumerate(self._template.get_stages())
                              if my_layer_index in stage._layer_indices)
        sampler: OobleckSampler = self._dataloader.batch_sampler
        self.train_schedule = OobleckPipelineSchedule(
            micro_batches=sampler.num_microbatches[self._pipeline_id],
            stages=len(self._template.get_stages()),
            stage_id=my_stage_index,
        )
        num_pipe_buffers = self.train_schedule.num_pipe_buffers()

        layer_cls = self._layer_cls
        if layer_cls is None:
            from .layer import Layer as layer_cls   # noqa: N813  (needs the CUDA extension; fails loudly otherwise)
        mb = self._training_args.per_device_train_batch_size
        workspace = layer_cls.make_workspace(model, mb, self.device) if hasattr(layer_cls, "make_workspace") else None

        layers = []
        shard_id = -1
        for layer_id, pg in self._per_layer_pgs.items():
            idx = pg.rank_index()
            if idx < 0:
                continue
            shard_id = idx
            if existing_pipeline is not None and existing_pipeline.execution is not None:   # :509-520
                existing_layer = next((l for l in existing_pipeline.execution._layers if l.layer_id == layer_id), None)
                if existing_layer is not None:
                    # a reused layer keeps its weights, moments and step count; if the new schedule is deeper its
                    # activation contexts are grown in place (a rebuilt Layer would restart from init_flat())
                    try:
                        layers.append(layer_cls.create_layer_from_layer(existing_layer, pg, num_pipe_buffers))
                    except TypeError:   # layer classes with the reference's two-argument signature
                        layers.append(layer_cls.create_layer_from_layer(existing_layer, pg))
                    continue
            extra = {}
            if existing_pipeline is not None and getattr(layer_cls, "supports_deferred_init", False):
                extra["init_values"] = False      # a layer that appears during a reconfiguration receives its state
            columns = len(self.rank_grid[layer_id])
            if columns > 1:
                if not getattr(layer_cls, "supports_sharding", False):
                    raise NotImplementedError(f"{layer_cls.__name__} cannot hold {columns} shard columns")
                extra["columns"] = columns
            layers.append(layer_cls(layer_id, model.layers[layer_id], pg, None, None, microbatch_size=mb,
                                    num_pipe_buffers=num_pipe_buffers, workspace=workspace, nsplit=self._nsplit,
                                    **extra))
        self.execution = PipelineExecution(pipeline=self, layers=layers, shard_id=shard_id,
                                           dataloader=self._dataloader, training_args=self._training_args)
        self.pipe_buffers: dict[str, list] = {
            "inputs": [None for _ in range(num_pipe_buffers)],    # batch input and received activations
            "labels": [None for _ in range(num_pipe_buffers)],    # labels from batch input
            "outputs": [None for _ in range(num_pipe_buffers)],   # activations to be sent
        }

    def is_first_stage(self) -> bool:
        return self.communication.prev_rank is None

    def is_last_stage(self) -> bool:
        return self.communication.next_rank is None
