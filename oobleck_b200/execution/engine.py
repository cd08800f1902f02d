"""Engine layer above the pipeline: data-parallel gradient all-reduce, reconfiguration, the training loop.

Mirrors oobleck/execution/engine.py:

    DataParallelEngine       :363-412  per-(layer, fsdp_index) groups over heterogeneous pipelines, SUM all-reduce
    ReconfigurationEngine    :39-360   rank re-assignment policy (borrow / merge) + state copy after a loss
    OobleckEngine            :415-668  construct -> initialize_distributed -> instantiate_pipelines -> train

The policy code (which ranks go where) is bit-exact with the reference (golden vectors from the reference's own
``on_reconfigure``; tests/test_engine_bookkeeping.py).  The *mechanism* is what changed:
* DP communicators are created once per distinct rank set instead of once per (layer, fsdp_index)
  (engine.py:390-392 issues O(layers) collective ``new_group`` calls on every rank);
* pipelines are rebuilt without tearing down the world process group and without per-layer groups;
* the planner (csrc/planning, planning/instantiator.py) is control plane and not part of this package: templates
  are injected (``templates=``) or derived with ``planning.pipeline_template.balanced_template``.
"""
from __future__ import annotations

import copy
import datetime
import math
import os
import queue
import socket
import threading
import time
import weakref
from collections import defaultdict
from dataclasses import dataclass, field
from typing import Any

import torch
import torch.distributed as dist

from ..module.model import OobleckModel
from ..planning.pipeline_template import PipelineTemplate, balanced_template
from .dataloader import LoaderType, OobleckDataLoader, SyntheticTokenDataset
from .pipeline import OobleckPipeline, PipelineAborted, RankGroup, bump_generation, run_interruptible
from .training_args import TrainingArguments


# ---- arguments (oobleck/elastic/training_util.py:7-39, plain dataclasses) ------------------------------------------
@dataclass
class DistributedArguments:
    master_ip: str = "127.0.0.1"
    master_port: int = 0
    node_ips: list[str] = field(default_factory=list)
    node_port: int = 22
    num_workers: int = 1
    num_agents_per_node: int = 1
    username: str | None = None


@dataclass
class JobArguments:
    fault_threshold: int = 3
    microbatch_size: int = 8
    global_microbatch_size: int = 128
    steps: int = 50
    eval_microbatch_size: int = 8      # sequences per evaluation micro-batch (HF per_device_eval_batch_size)


@dataclass
class ModelArguments:
    model_name: str = "gpt2"
    model_tag: str = "small"
    dataset_path: str = "wikitext"
    dataset_name: str | None = "wikitext-2-raw-v1"
    model_args: dict[str, Any] = field(default_factory=dict)


@dataclass
class OobleckArguments:
    dist: DistributedArguments = field(default_factory=DistributedArguments)
    job: JobArguments = field(default_factory=JobArguments)
    model: ModelArguments = field(default_factory=ModelArguments)


@dataclass
class DistributionInfo:
    """What the agent sends once on the worker pipe (oobleck/elastic/message_util.py:11-13).  The engine only reads
    ``agent_ips`` and ``world_size``: the control plane's own class is accepted as is (duck typing)."""
    agent_ips: list[str]
    world_size: int


def _rank() -> int:
    return dist.get_rank() if dist.is_initialized() else 0


_DEBUG = os.environ.get("OOB_ELASTIC_DEBUG", "0") == "1"


def _dbg(msg: str) -> None:
    if _DEBUG:
        import sys
        print(f"[elastic rank {_rank()} {time.perf_counter():.3f}] {msg}", file=sys.stderr, flush=True)


def _my_ip() -> str:
    """engine.py:555 (``socket.gethostbyname(socket.gethostname())``; the reference's tests patch it)."""
    try:
        return socket.gethostbyname(socket.gethostname())
    except OSError:
        return "127.0.0.1"


# Communicators survive pipeline rebuilds: one per rank set for the life of the process.  (torch names group-local
# groups by a hash of their ranks, so creating the same set twice would also collide in the rendezvous store.)
_COMMUNICATORS: dict[tuple[int, ...], Any] = {}


_GROUP_CREATIONS: dict[tuple[int, ...], int] = {}


def _new_member_group(ranks, timeout=None):
    """``dist.new_group(ranks, use_local_synchronization=True)`` -- only the member ranks take part, which is what lets
    survivors build communicators after a loss -- with a rendezvous name every member derives identically.  torch
    hashes the rank list together with ``len(_world.pg_names)``, the number of groups THIS process has created so far
    (distributed_c10d._hash_ranks_to_str); after a reconfiguration that count differs between members (they belonged to
    different groups before) and their rendezvous keys never meet.  The name used here is the rank set plus how many
    times this very set has been created -- every member has taken part in each of those creations."""
    import hashlib

    import torch.distributed.distributed_c10d as c10d
    key = tuple(sorted(ranks))
    n = _GROUP_CREATIONS[key] = _GROUP_CREATIONS.get(key, 0) + 1
    name = hashlib.sha1(("oobleck_b200_" + "_".join(map(str, key)) + f"#{n}").encode(), usedforsecurity=False).hexdigest()
    kw = {} if timeout is None else {"timeout": timeout}
    orig = getattr(c10d, "_hash_ranks_to_str", None)
    if orig is None:
        return dist.new_group(list(key), use_local_synchronization=True, **kw)
    c10d._hash_ranks_to_str = lambda _ranks: name
    try:
        return dist.new_group(list(key), use_local_synchronization=True, **kw)
    finally:
        c10d._hash_ranks_to_str = orig


def _communicator(ranks, timeout):
    """The process-wide communicator of the rank set ``ranks`` (any order), created on first use."""
    key = tuple(sorted(ranks))
    if key not in _COMMUNICATORS:
        _COMMUNICATORS[key] = _new_member_group(key, timeout)
    return _COMMUNICATORS[key]


def _moved_state(layer) -> list[torch.Tensor]:
    """What moves when a layer changes owner: ``state_tensors()`` and its AdamW step count as a one-element int64
    tensor on the same device."""
    return list(layer.state_tensors()) + [torch.tensor([layer.opt_step], dtype=torch.int64,
                                                       device=layer.flat_param.device)]


# ---- data parallel -------------------------------------------------------------------------------------------------
class DataParallelEngine:
    def __init__(self, engine, pipelines: list[OobleckPipeline], new_group=None):
        self._engine = weakref.ref(engine)
        # layer_index -> fsdp_index -> ranks (engine.py:374-384)
        ranks_grid: dict[int, dict[int, list[int]]] = defaultdict(dict)
        for pipeline in pipelines:
            for layer_index, ranks in pipeline.rank_grid.items():
                assert isinstance(ranks, list) and len(ranks) == engine._num_gpus_per_node
                for fsdp_index, rank in enumerate(ranks):
                    ranks_grid[layer_index].setdefault(fsdp_index, []).append(rank)
        self._ranks_grid = ranks_grid
        self._comm_stream = None
        self._pending: list = []
        self._overlapped: set[int] = set()
        # One communicator per DISTINCT rank set, created in first-use order (identical on every rank).  The reference
        # calls new_group once per (layer, fsdp_index) (:390-392); the mapping below is otherwise the same.
        my_rank = _rank()

        def _make(ranks):
            # group-local creation: only member ranks take part, so survivors can build communicators after a loss
            # without re-creating the world group (engine.py:539-593 tears the NCCL world down and re-inits it)
            if not dist.is_initialized() or len(ranks) <= 1 or my_rank not in ranks:
                return None
            return _communicator(ranks, engine._comm_timeout)

        make = new_group or _make
        cache: dict[tuple[int, ...], Any] = {}
        self._dp_process_groups: dict[int, dict[int, RankGroup]] = defaultdict(dict)
        self._fsdp_indices: dict[int, list[int]] = defaultdict(list)
        self.group_creation_order: list[list[int]] = []
        for layer_index, per_layer in ranks_grid.items():
            for fsdp_index, ranks in per_layer.items():
                key = tuple(ranks)
                if key not in cache:
                    cache[key] = make(list(ranks))
                    self.group_creation_order.append(list(ranks))
                self._dp_process_groups[layer_index][fsdp_index] = RankGroup(list(ranks), my_rank, cache[key])
                if my_rank in ranks:
                    self._fsdp_indices[layer_index].append(fsdp_index)

    @property
    def engine(self):
        return self._engine()

    def _groups_of(self, layer):
        process_groups = {fi: pg for fi, pg in self._dp_process_groups[layer.layer_id].items() if pg.rank_index() >= 0}
        if process_groups and any(pg.size() > 1 for pg in process_groups.values()):
            return process_groups
        return None

    def touches(self, ranks: set[int]) -> bool:
        """Does any communicator this rank reduces gradients over contain one of ``ranks``?"""
        if not ranks:
            return False
        for layer in self.engine._pipeline.execution._layers:
            for pg in (self._groups_of(layer) or {}).values():
                if ranks & set(pg.ranks):
                    return True
        return False

    def layer_ready(self, layer):
        """Hook of ``PipelineExecution.backward_pass`` for the step's last micro-batch (non-elastic CUDA runs): the
        layer's gradient is complete once this backward and its side-stream weight-gradient kernels have run, so its
        SUM all-reduce starts now on the communication stream and overlaps the backward of the layers before it and
        the pipeline flush.  (The reference reduces layer by layer after the whole step, blocking:
        engine.py:404-412, layer.py:290-291.)  One bucket per layer: the flat gradient is already contiguous."""
        pgs = self._groups_of(layer)
        if pgs is None:
            if not layer.sharded:
                return
            pgs = {}       # no replica, but the stage shards the layer: its reduce-scatter starts now all the same
        import ctypes as C

        from .. import lib as L
        if self._comm_stream is None:
            self._comm_stream = torch.cuda.Stream()
        cs = self._comm_stream
        cs.wait_stream(torch.cuda.current_stream())
        L.call("oob_side_join", C.c_void_p(cs.cuda_stream))     # this layer's wgrad / bias-sum kernels
        with torch.cuda.stream(cs):
            self._pending.extend(layer.reduce_gradients(pgs, async_op=True))
        self._overlapped.add(layer.layer_id)

    def do_allreduce(self):
        """engine.py:404-412: every local layer reduces over the groups that contain this rank (SUM, never averaged).
        Layers whose reduction was started early by ``layer_ready`` are only waited for."""
        for layer in self.engine._pipeline.execution._layers:
            if layer.layer_id in self._overlapped:
                continue
            pgs = self._groups_of(layer)
            if pgs is not None:
                layer.reduce_gradients(pgs)
        for w in self._pending:
            w.wait()                          # the compute stream waits for the NCCL stream; the host does not block
        if self._overlapped and self._comm_stream is not None:
            # collectives that were already waited for on the communication stream itself (a sharded layer's
            # reduce-scatter, which its cross-replica all-reduce consumes there)
            torch.cuda.current_stream().wait_stream(self._comm_stream)
        self._pending.clear()
        self._overlapped.clear()


# ---- peer shadow ---------------------------------------------------------------------------------------------------
class PeerShadow:
    """Stage state mirrored on the neighbouring stage, so that a pipeline WITHOUT a replica survives the loss of a rank
    (BASELINE config 5: one 8-stage pipeline -> 7 stages; SURVEY 7 hard part 5, 8(f1)).  The reference cannot: every
    layer of the lost stage has "no alive ranks" and ``_copy_model_states`` raises (engine.py:263-269).

    Ring over the stages of one pipeline: the rank of stage ``s`` keeps a copy of everything stage ``s + 1`` would lose
    -- ``flat_param``, ``exp_avg``, ``exp_avg_sq`` and the AdamW step count of each of its layers -- refreshed after
    every committed optimizer step with one broadcast per layer inside the two-rank communicator of the pair (NVLink:
    GPT-2-XL on 8 stages moves ~2.2 GB per rank and step, a few milliseconds next to a step of about a second).
    After a loss the holder sends the shadow to whoever owns those layers in the new pipeline."""

    def __init__(self, engine, pipeline: OobleckPipeline):
        self._engine = weakref.ref(engine)
        stages = pipeline._template.get_stages()
        self.stage_ranks = [pipeline.rank_grid[st._layer_indices[0]][0] for st in stages]
        self.stage_layers = [list(st._layer_indices) for st in stages]
        P = len(self.stage_ranks)
        self.enabled = P > 1 and engine._num_gpus_per_node == 1
        self.holder_of_layer: dict[int, int] = {}
        self.held: dict[int, list[torch.Tensor]] = {}      # layer id -> [param, exp_avg, exp_avg_sq, step]
        self.staging: dict[int, list[torch.Tensor]] = {}   # where a refresh lands before it replaces ``held``
        self.last_refresh_ok = True
        self.groups: dict[tuple[int, int], Any] = {}
        if not self.enabled:
            return
        me = engine._rank
        for s in range(P):
            for l in self.stage_layers[s]:
                self.holder_of_layer[l] = self.stage_ranks[(s - 1) % P]
        device = pipeline.device
        for s in range(P):                                   # same creation order on both members of a pair
            a, b = self.stage_ranks[(s - 1) % P], self.stage_ranks[s]      # holder, owner
            if me in (a, b):
                self.groups[(a, b)] = _communicator((a, b), engine._comm_timeout)
            if me == a:
                for l in self.stage_layers[s]:
                    n = engine._model.layers[l].num_params
                    self.held[l] = [torch.zeros(n, dtype=torch.float32, device=device) for _ in range(3)] + \
                                   [torch.zeros(1, dtype=torch.int64, device=device)]

    def refresh(self):
        """After a committed optimizer step: owners publish, holders receive (all broadcasts asynchronous, then waited:
        every rank is a source in one pair and a destination in another).

        The mirror changes atomically: a holder receives into a second set of buffers and swaps the two sets only when
        every tensor of the mirrored stage has arrived.  Arrival is judged by the step count, the LAST tensor broadcast
        for a layer on the pair's communicator (collectives of one communicator complete in order): the receive buffer
        is preset to -1 and must come back as one non-negative count, the same for every layer of the stage.  An owner
        that dies in here (gloo: the wait raises; NCCL: the listener aborts the communicator and the count never
        arrives) leaves the mirror exactly as the previous step left it."""
        if not self.enabled:
            return
        engine = self._engine()
        me = engine._rank
        works = []
        P = len(self.stage_ranks)
        mine = engine._pipeline.execution._layers
        receiving: list[int] = []
        for s in range(P):
            a, b = self.stage_ranks[(s - 1) % P], self.stage_ranks[s]
            if me == b:
                for layer in mine:
                    if layer.layer_id in self.stage_layers[s]:
                        for t in _moved_state(layer):
                            works.append(dist.broadcast(t, src=b, group=self.groups[(a, b)], async_op=True))
            if me == a:
                for l in self.stage_layers[s]:
                    if l not in self.staging:
                        self.staging[l] = [torch.zeros_like(t) for t in self.held[l]]
                    self.staging[l][3].fill_(-1)
                    receiving.append(l)
                    for t in self.staging[l]:
                        works.append(dist.broadcast(t, src=b, group=self.groups[(a, b)], async_op=True))
        failed = False
        for w in works:
            try:
                w.wait()
            except RuntimeError:
                failed = True
        if receiving and not failed:
            try:
                counts = {int(self.staging[l][3].item()) for l in receiving}
                failed = len(counts) != 1 or min(counts) < 0
            except RuntimeError:
                failed = True
        if receiving and not failed:
            for l in receiving:
                self.held[l], self.staging[l] = self.staging[l], self.held[l]
        self.last_refresh_ok = not failed


# ---- reconfiguration -----------------------------------------------------------------------------------------------
class ReconfigurationEngine:
    def __init__(self, engine, pipelines: list[OobleckPipeline], start_listener: bool = True):
        self._engine = weakref.ref(engine)
        self._pipelines = pipelines
        self._num_instances_set: dict[PipelineTemplate, int] = defaultdict(int)
        for pipeline in self._pipelines:
            self._num_instances_set[pipeline._template] += 1
        t0 = engine._pipeline_templates[0]
        self._min_num_ranks = t0._num_nodes * t0._num_gpus_per_node          # engine.py:46-49
        self.last_reconfiguration_seconds: float | None = None
        self.last_breakdown: dict | None = None
        self.last_notification_time: float | None = None
        # lost-rank lists received by the listener thread, applied by the training thread at its next safe point
        self._pending: "queue.Queue[tuple[list[int], float]]" = queue.Queue()
        self._reconfiguration_listener = None
        if start_listener and getattr(engine, "_agent_pipe", None) is not None and engine._listen:
            self._reconfiguration_listener = threading.Thread(target=self._reconfiguration_listener_fn, daemon=True)
            self._reconfiguration_listener.start()

    @property
    def engine(self):
        return self._engine()

    def _reconfiguration_listener_fn(self):
        """Daemon thread (engine.py:50-61).  The reference rebuilds the pipelines from this thread while the training
        thread is inside a step, with no lock; here the listener only does what cannot wait -- the pipe round trip and
        releasing every stream / communicator that is stuck on the lost ranks -- and hands the re-planning to the
        training thread (``poll``), which applies it between two steps."""
        while True:
            try:
                engine = self.engine
                if engine is None:
                    return
                lost_node: str = engine._agent_pipe.recv()
            except (EOFError, ValueError, OSError):
                return                                          # connection closed (engine.py:78-80)
            t0 = time.perf_counter()
            _dbg(f"listener: lost node {lost_node}")
            try:
                lost_ranks = self.remove_lost_node_from_dist_info(lost_node)
                engine.on_ranks_lost(lost_ranks)                # first: un-wedge the GPU
                engine.initialize_distributed()                 # port round trip with the agent (engine.py:572-578)
            except (EOFError, ValueError, OSError):
                return
            _dbg(f"listener: queued reconfiguration for lost ranks {lost_ranks}")
            self._pending.put((lost_ranks, t0))

    def poll(self) -> bool:
        """Training thread: apply every reconfiguration the listener has queued.  True if the pipelines changed."""
        changed = False
        while True:
            try:
                lost_ranks, t0 = self._pending.get_nowait()
            except queue.Empty:
                return changed
            self.last_notification_time = t0
            _dbg(f"poll: reconfiguring for lost ranks {lost_ranks}")
            self.on_reconfigure(lost_ranks)
            self.last_reconfiguration_seconds = time.perf_counter() - t0
            _dbg(f"poll: done in {self.last_reconfiguration_seconds:.3f}s")
            self.engine._notified = not self._pending.empty()
            changed = True

    def _on_receive_reconfiguration_notification(self) -> bool:
        """engine.py:63-80, synchronous form (the reference's tests call it directly,
        tests/execution/test_engine.py:967-1019).  Returns False when the agent pipe is closed."""
        try:
            engine = self.engine
            lost_node: str = engine._agent_pipe.recv()
            t0 = time.perf_counter()
            lost_ranks = self.remove_lost_node_from_dist_info(lost_node)
            engine.on_ranks_lost(lost_ranks)
            engine.initialize_distributed()
            self.last_notification_time = t0
            self.on_reconfigure(lost_ranks)
            self.last_reconfiguration_seconds = time.perf_counter() - t0
            engine._notified = False
            return True
        except (EOFError, ValueError, OSError):
            return False

    def remove_lost_node_from_dist_info(self, lost_node_ip: str) -> list[int]:   # engine.py:82-89
        engine = self.engine
        assert getattr(engine, "_dist_info", None) is not None, "Distributed is not initialized yet."
        engine._dist_info.agent_ips.remove(lost_node_ip)
        engine._dist_info.world_size -= engine._num_gpus_per_node
        return engine._rank_map.pop(lost_node_ip)

    # -- policy (bit-exact with engine.py:91-166, 311-360) -----------------------------------------------------------
    def plan_new_ranks(self, lost_ranks: list[int]) -> list[list[int]]:
        for pipeline in self._pipelines:
            pipeline._ranks = [rank for rank in pipeline._ranks if rank not in lost_ranks]
        need_merge = False
        new_ranks_list: list[list[int]] = []
        for pipeline in self._pipelines:
            ranks = pipeline._ranks
            if len(ranks) == 0:
                continue                              # every rank of this pipeline is gone
            if len(ranks) >= self._min_num_ranks:
                new_ranks_list.append(ranks)          # some template still fits
                continue
            while len(ranks) < self._min_num_ranks:   # borrow from the biggest pipeline
                biggest = self._find_biggest_pipeline(self._pipelines)
                if biggest is None:
                    need_merge = True
                    break
                while len(biggest._ranks) > self._min_num_ranks and len(ranks) < self._min_num_ranks:
                    ranks.append(biggest._ranks.pop())
            new_ranks_list.append(ranks)
        if need_merge:
            new_ranks_list = self._merge_pipelines(new_ranks_list)
        for ranks in new_ranks_list:
            ranks.sort()
        new_ranks_list.sort(key=lambda ranks: (len(ranks), ranks[0]))
        return new_ranks_list

    def _merge_pipelines(self, ranks_list: list[list[int]]) -> list[list[int]]:
        to_merge = [r for r in ranks_list if len(r) < self._min_num_ranks]
        results = [r for r in ranks_list if len(r) >= self._min_num_ranks]
        try:
            while to_merge:
                ranks = to_merge.pop(0)
                try:
                    while len(ranks) < self._min_num_ranks:
                        ranks.extend(to_merge.pop(0))
                except IndexError:
                    ranks.extend(results.pop(0))      # nothing small left: absorb the first healthy pipeline
                assert len(ranks) >= self._min_num_ranks
                results.append(ranks)
        except IndexError:
            raise RuntimeError("Ranks are insufficient")
        return results

    def _find_biggest_pipeline(self, pipelines):
        biggest = None
        for pipeline in pipelines:
            if biggest is None or len(pipeline._ranks) >= len(biggest._ranks):
                biggest = pipeline
        if biggest is not None and len(biggest._ranks) > self._min_num_ranks:
            return biggest
        return None

    def on_reconfigure(self, lost_ranks: list[int]):
        def get_pipeline_template(ranks, templates):
            return next((t for t in templates if t._num_nodes * t._num_gpus_per_node == len(ranks)), None)

        t_phase = [time.perf_counter()]
        old_rank_grids = [copy.deepcopy(pipeline.rank_grid) for pipeline in self._pipelines]
        new_ranks_list = self.plan_new_ranks(lost_ranks)
        new_num_instances_set: dict[PipelineTemplate, int] = defaultdict(int)
        for ranks in new_ranks_list:
            new_num_instances_set[get_pipeline_template(ranks, self.engine._pipeline_templates)] += 1
        new_pipeline = self._reinstantiate(new_num_instances_set, new_ranks_list)
        t_phase.append(time.perf_counter())
        new_rank_grids = []
        remaining = list(new_ranks_list)
        for template, num_instance in new_num_instances_set.items():
            for _ in range(num_instance):
                new_rank_grids.append(template.get_rank_grid(remaining.pop(0)))
        self._copy_model_states(old_rank_grids, new_rank_grids, new_pipeline)
        t_phase.append(time.perf_counter())
        for layer in self.engine._pipeline.execution._layers:        # engine.py:176-178
            if all(layer is not l for l in new_pipeline.execution._layers):
                layer.remove_tensors()
        self.engine._pipeline = new_pipeline
        self.engine._install_dp_overlap()
        self.engine._make_job_group()
        if self.engine._peer_shadow:
            self.engine._shadow = PeerShadow(self.engine, new_pipeline)
            self.engine._shadow.refresh()
        t_phase.append(time.perf_counter())
        self.last_breakdown = {"plan_and_rebuild_pipelines_s": t_phase[1] - t_phase[0],
                               "copy_model_states_s": t_phase[2] - t_phase[1],
                               "communicators_and_shadows_s": t_phase[3] - t_phase[2]}

    # -- mechanism ---------------------------------------------------------------------------------------------------
    def _reinstantiate(self, num_instances_set, new_ranks_list) -> OobleckPipeline:
        engine = self.engine
        bump_generation()     # wire traffic of the new pipelines can never match a receive abandoned by the old ones
        global_num_microbatch = engine._args.job.global_microbatch_size // engine._args.job.microbatch_size
        templates = [t for t, n in num_instances_set.items() for _ in range(n)]
        num_microbatches = engine.distribute_microbatches(templates, global_num_microbatch)
        my_index = next(i for i, ranks in enumerate(new_ranks_list) if engine._rank in ranks)
        sampler = engine._pipeline._dataloader.batch_sampler
        dataloader = OobleckDataLoader(engine._hf_training_args, engine._dataset, LoaderType.Training, my_index,
                                       num_microbatches, sampler.num_iterations_done, sampler.epoch,
                                       device_resident=engine._device_resident)
        pipelines, mine = [], None
        for pid, (template, ranks) in enumerate(zip(templates, new_ranks_list)):
            p = engine.make_pipeline(pid, template, list(ranks), dataloader, engine._pipeline._global_step)
            pipelines.append(p)
            if p.my_pipeline:
                mine = p
        for p in pipelines:
            p.initialize_distributed_fsdp()
            p.initialize_distributed_pipeline()
        mine.initialize_execution(engine._model, engine._pipeline)
        engine._dp_engine = DataParallelEngine(engine, pipelines)
        self._pipelines = pipelines
        return mine

    def _copy_model_states(self, old_rank_grids, new_rank_grids, new_pipeline: OobleckPipeline):
        """engine.py:238-309: per layer, some old owner whose rank list survives unchanged sends the layer to the new
        owners.  Same sender choice and the same RuntimeError; the transfer itself is a broadcast inside the (cached)
        DP communicator of that layer.  Beyond the reference (which moves ``flat_param`` only and lets the moved
        layer's Adam moments restart from zero): ``exp_avg``, ``exp_avg_sq`` and the layer's AdamW step count travel
        too, so every replica of a layer holds the same optimizer state after the move."""
        engine = self.engine
        works = []
        for layer_index in range(len(old_rank_grids[0])):
            old_ranks = [g[layer_index] for g in old_rank_grids]
            new_ranks = [g[layer_index] for g in new_rank_grids]
            if all(rank in old_ranks for rank in new_ranks):
                continue
            alive = [ranks for ranks in old_ranks if ranks in new_ranks]
            my_rank = engine._rank if dist.is_initialized() else _rank()
            if not alive:
                # Nobody keeps this layer in place.  The reference gives up here (engine.py:263-269).  With peer
                # shadows a source still exists: an old owner that survived (the layer merely moves to another stage of
                # the re-split pipeline), else the neighbour that mirrors the lost stage.
                moved = self._move_without_replica(layer_index, old_ranks, new_ranks, new_pipeline, my_rank)
                if moved is None:
                    raise RuntimeError(f"No alive ranks for the layer {layer_index}. Terminating.")
                works.extend(moved)
                continue
            ranks_to_send = alive[0]
            for ranks_recv in new_ranks:
                if my_rank not in ranks_recv:
                    continue
                fsdp_index = ranks_recv.index(my_rank)
                dp_group = engine._dp_engine._dp_process_groups[layer_index][fsdp_index]
                new_layer = next(l for l in new_pipeline.execution._layers if l.layer_id == layer_index)
                src = ranks_to_send[fsdp_index]
                if my_rank == src:
                    old_layer = next(l for l in engine._pipeline.execution._layers if l.layer_id == layer_index)
                    if new_layer is not old_layer:
                        if hasattr(new_layer, "adopt_state_"):
                            new_layer.adopt_state_(old_layer)
                        else:
                            new_layer.load_flat_(old_layer.flat_param)
                if dp_group.group is not None:
                    tensors = _moved_state(new_layer)
                    step = tensors[-1]
                    for t in tensors:
                        works.append((dist.broadcast(t, src=src, group=dp_group.group, async_op=True), new_layer,
                                      step if t is step else None))
        for work, layer, step in works:
            if work is not None:
                work.wait()
            if step is not None and layer is not None:
                layer.opt_step = int(step.item())
                layer.refresh_planes()
        # no world barrier (engine.py:308): a lost rank can never join it; the broadcasts above are the only ordering
        if torch.cuda.is_available():
            torch.cuda.synchronize()


    def _move_without_replica(self, layer_index, old_ranks, new_ranks, new_pipeline, my_rank):
        """Source = a surviving old owner of the layer, else its peer shadow; destinations = its new owners.  Returns the
        list of (work, layer, step) entries ``_copy_model_states`` waits on, or None when no source exists."""
        engine = self.engine
        shadow = getattr(engine, "_shadow", None)
        lost = getattr(engine, "_lost_ranks", set())
        if shadow is None and not getattr(engine, "_peer_shadow", False):
            return None          # reference behaviour: a layer nobody keeps in place is unrecoverable
        old_owners = [r[0] for r in old_ranks]
        src = next((r for r in old_owners if r not in lost), None)
        from_shadow = False
        if src is None:
            if shadow is None or not shadow.enabled or layer_index not in shadow.holder_of_layer:
                return None
            src = shadow.holder_of_layer[layer_index]
            if src in lost:
                return None                     # the stage and the neighbour holding its mirror died together
            from_shadow = True
        dsts = [r[0] for r in new_ranks]
        members = tuple(sorted(set([src] + dsts)))
        out = []
        if my_rank not in members:
            return out
        new_layer = next((l for l in new_pipeline.execution._layers if l.layer_id == layer_index), None)
        if my_rank == src:
            if from_shadow:
                tensors = shadow.held[layer_index]
            else:
                old_layer = next(l for l in engine._pipeline.execution._layers if l.layer_id == layer_index)
                tensors = _moved_state(old_layer)
            if new_layer is not None and my_rank in dsts:      # the source is one of the new owners: local copy
                for dst_t, src_t in zip(new_layer.state_tensors(), tensors[:3]):
                    dst_t.copy_(src_t)
                out.append((None, new_layer, tensors[3].clone()))
        else:
            tensors = _moved_state(new_layer)     # receive buffers: every value is overwritten by the broadcast
        if len(members) > 1:
            group = _communicator(members, engine._comm_timeout)
            for i, t in enumerate(tensors):
                w = dist.broadcast(t, src=src, group=group, async_op=True)
                is_step = i == len(tensors) - 1
                if my_rank != src:
                    out.append((w, new_layer, t if is_step else None))
                else:
                    out.append((w, None, None))
        return out


# ---- engine --------------------------------------------------------------------------------------------------------
def layer_cost_model(model: OobleckModel, microbatch: int) -> list[float]:
    """Relative fwd+bwd cost per stage layer (FLOPs): stand-in for the profiler's per-layer latencies
    (planning/profiler.py:41-123), used only to balance stages when no planner template is injected."""
    costs = []
    for spec in model.layers:
        E, T, V = spec.n_embd, spec.n_positions, spec.vocab_size
        if spec.kind == "block":
            costs.append(6.0 * 12 * E * E + 12.0 * T * E * 0.5)
        elif spec.kind == "head":
            costs.append(6.0 * E * V)
        else:
            costs.append(1e-3 * E)
    return costs


def node_range(profile_results, num_nodes: int, num_gpus_per_node: int, device_memory_bytes: int) -> tuple[int, int]:
    """``(min_num_nodes, max_num_nodes)`` handed to ``create_pipeline_templates`` -- engine.py:490-514, same arithmetic
    and the same assertion text (golden table: tests/execution/test_engine.py:394-406).  A pipeline needs six copies of
    every layer's parameter bytes (weights, gradients, optimizer state, ...) plus the largest single activation
    footprint; the minimum node count is that total over the memory of one node's GPUs, at least 1."""
    import math
    layers = profile_results.get()
    total_memory_consumption = 6 * sum(r._mem_required[0] for r in layers)
    total_memory_consumption += max(r._mem_required[1] for r in layers)
    min_num_nodes = max(1, math.ceil(total_memory_consumption / (device_memory_bytes * num_gpus_per_node)))
    max_num_nodes = num_nodes
    assert min_num_nodes <= max_num_nodes, (
        "Minimum required number of nodes is larger than maximum number of nodes "
        f"(minimum required: {min_num_nodes}, you have: {max_num_nodes})."
    )
    return min_num_nodes, max_num_nodes


class OobleckEngine:
    """engine.py:415-668.  ``pipe`` is the agent connection (may be None when launched by torchrun; rank/world then
    come from the environment)."""

    def __init__(self, local_rank: int, num_nodes: int, num_gpus_per_node: int, pipe, args: OobleckArguments, *,
                 dataset=None, templates: list[PipelineTemplate] | None = None, nsplit: int = 3, layer_cls=None,
                 transport_cls=None, device_resident: bool = False, listen: bool = True, backend: str | None = None,
                 comm_timeout_s: float | None = None, peer_shadow: bool | None = None):
        self._agent_pipe = pipe
        if pipe is not None:
            # elastic run: a dead peer is this engine's business (listener thread: abort + reconfigure), not the NCCL
            # watchdog's, which would tear the whole process down on the first remote error
            os.environ.setdefault("TORCH_NCCL_ASYNC_ERROR_HANDLING", "0")
        # mirror every stage's state on its neighbour (PeerShadow): off by default -- it only matters for pipelines
        # without a replica -- OOB_PEER_SHADOW=1 or peer_shadow=True turns it on
        self._peer_shadow = (os.environ.get("OOB_PEER_SHADOW", "0") == "1") if peer_shadow is None else bool(peer_shadow)
        self._shadow = None
        # timeout of every communicator this engine creates (None: torch's default); a replica that waits in an
        # all-reduce for a partner that dropped the step is released by ``on_ranks_lost`` (NCCL) or by this timeout
        self._comm_timeout = None if comm_timeout_s is None else datetime.timedelta(seconds=comm_timeout_s)
        self._listen = listen            # start the reconfiguration listener thread (engine.py:50-53) when a pipe exists
        self._backend = backend          # None: nccl on GPUs, gloo on CPU
        self._dist_info = None
        self._rank_map: dict[str, list[int]] = {}
        self._store = None
        self._store_port: int | None = None
        self._reconfigured = False
        self._lost_ranks: set[int] = set()
        self._job_group = None
        self._job_ranks: list[int] = []
        self._notified = False           # a loss notification has arrived and has not been applied yet
        self._args = args
        self._hf_training_args = TrainingArguments(per_device_train_batch_size=args.job.microbatch_size,
                                                   per_device_eval_batch_size=args.job.eval_microbatch_size,
                                                   max_steps=args.job.steps)
        self._local_rank = local_rank
        self._num_nodes = num_nodes
        self._num_gpus_per_node = num_gpus_per_node
        self._nsplit = nsplit
        self._layer_cls = layer_cls
        self._transport_cls = transport_cls
        self._device_resident = device_resident
        self._rank = 0
        self._world_size = num_nodes * num_gpus_per_node
        self.step_seconds: list[float] = []
        self.step_end_times: list[float] = []     # time.perf_counter() at the end of every completed step
        self._reconfiguration = None
        self._step_aborted = False

        margs = dict(args.model.model_args)
        n_positions = margs.get("n_positions", 1024)
        self._model = OobleckModel(args.model.model_name, {"input_ids": None, "attention_mask": None, "labels": None},
                                   self._hf_training_args, args.model.model_tag, margs)
        self._dataset = dataset if dataset is not None else SyntheticTokenDataset(
            seq_len=n_positions, vocab_size=self._model.model_args.vocab_size)
        # Without injected templates (the planner is control plane) stages are balanced on per-layer costs: measured
        # on the GPU at instantiate_pipelines() time when this engine runs CUDA layers (planning/profiler.py), from the
        # FLOP model otherwise.  ``layer_costs`` is kept for inspection (bench.py prints it).
        self.layer_costs: list[float] | None = None
        self.layer_costs_source = "FLOP model"
        self._templates_injected = templates is not None
        if templates is None:
            self.layer_costs = layer_cost_model(self._model, args.job.microbatch_size)
            templates = [balanced_template(self.layer_costs, n, num_gpus_per_node)
                         for n in range(1, num_nodes + 1) if n <= len(self.layer_costs)]
        self._pipeline_templates = templates

    # -- distributed -------------------------------------------------------------------------------------------------
    def initialize_distributed(self, backend: str | None = None):
        """engine.py:526-596.  With an agent pipe the reference's protocol is followed message for message:

            first call : recv DistributionInfo; rank 0 (first agent IP, local rank 0) creates TCPStore(port=0),
                         sends the port up the pipe and discards the agent's echo; everyone else receives the port
            later calls: (after a lost-node notification) the same port round trip, so the agent's pipe stays in step

        What differs is what happens around it: the reference destroys the NCCL world here and re-creates it on every
        reconfiguration (:532-540, :588-593); this engine keeps the world it built on the first call -- ranks keep
        their numbers (``_rank_map`` is only popped, like the reference's) and survivors talk over communicators that
        never contained the lost ranks.  Without a pipe (torchrun launch) rank / world come from the environment."""
        backend = backend or self._backend or ("nccl" if torch.cuda.is_available() else "gloo")
        if self._agent_pipe is None:
            if dist.is_initialized():
                self._rank, self._world_size = dist.get_rank(), dist.get_world_size()
                return
            world = int(os.environ.get("WORLD_SIZE", "1"))
            if world > 1:
                dist.init_process_group(backend=backend)
                self._rank, self._world_size = dist.get_rank(), dist.get_world_size()
            else:
                self._rank, self._world_size = 0, 1
            return

        pipe = self._agent_pipe
        if self._dist_info is None:
            self._dist_info = pipe.recv()                                              # engine.py:543
            self._rank_map = {ip: list(range(i * self._num_gpus_per_node, (i + 1) * self._num_gpus_per_node))
                              for i, ip in enumerate(self._dist_info.agent_ips)}       # :544-552
        dist_info = self._dist_info
        my_ip = _my_ip()
        assert my_ip in dist_info.agent_ips, f"My IP {my_ip} is not in dist info {dist_info.agent_ips}."
        self._num_nodes = len(dist_info.agent_ips)
        self._world_size = dist_info.world_size
        self._rank = self._rank_map[my_ip][self._local_rank]
        is_master = next(iter(self._rank_map)) == my_ip and self._local_rank == 0      # :563

        if dist.is_initialized():
            # reconfiguration: the world stays; only the agent's port round trip is honoured (:572-578)
            if is_master:
                pipe.send(self._store_port if self._store_port is not None else 0)
                pipe.recv()
            else:
                pipe.recv()
            return
        if is_master:
            store = dist.TCPStore(host_name=my_ip, port=0, world_size=dist_info.world_size, is_master=True,
                                  wait_for_workers=False)
            self._store_port = store.port
            pipe.send(store.port)
            pipe.recv()            # the agent sends the port back to every worker, rank 0 included: discard it
        else:
            port: int = pipe.recv()
            self._store_port = port
            store = dist.TCPStore(host_name=dist_info.agent_ips[0], port=port, world_size=dist_info.world_size,
                                  is_master=False, wait_for_workers=False)
        self._store = store
        kw = {} if self._comm_timeout is None else {"timeout": self._comm_timeout}
        dist.init_process_group(backend=backend, store=store, rank=self._rank, world_size=dist_info.world_size, **kw)
        assert dist.is_initialized()

    def on_ranks_lost(self, lost_ranks: list[int]):
        """Release everything on this rank that is (or would get) stuck on a lost rank.  Callable from the listener
        thread while the training thread is inside a step:

        * inter-stage links: ``transport.abort()`` writes the abort word of every mailbox through host-mapped memory, so
          send / recv kernels spinning on a dead neighbour return at once (otherwise: the 120 s watchdog of
          csrc/p2p.cu);
        * cross-replica communicators that contain a lost rank are aborted (``ncclCommAbort`` under
          ``ProcessGroup.abort``) and dropped from the cache; survivors get fresh ones in ``DataParallelEngine``.

        The reference has no counterpart: it destroys the whole NCCL world from the listener thread (engine.py:532-540)
        and notes that this may hang when a collective is in flight."""
        lost = set(lost_ranks)
        self._reconfigured = True
        self._lost_ranks |= lost
        self._notified = True
        # my stage may be waiting for a neighbour that is lost -- or alive but already dropping the step: release it
        pipeline = getattr(self, "_pipeline", None)
        if pipeline is not None and pipeline.communication is not None:
            pipeline.communication.transport.abort()
        # communicators that contain a lost rank can never complete anything again
        for key in [k for k in _COMMUNICATORS if lost & set(k)]:
            group = _COMMUNICATORS.pop(key)
            try:
                if hasattr(group, "abort") and dist.get_backend(group) == "nccl":
                    group.abort()          # ncclCommAbort: releases kernels blocked on the dead peer
            except Exception:  # noqa: BLE001  (gloo cannot abort; an op on a dead peer ends with a peer-reset error)
                pass

    # -- planning stand-ins ------------------------------------------------------------------------------------------
    def _install_dp_overlap(self):
        """Overlapped all-reduce only where it is safe: CUDA layers, replicas exist, and no agent pipe (an elastic step
        must not exchange gradients before its vote -- ``_guarded_train_step``)."""
        ex = self._pipeline.execution
        overlap = (self._agent_pipe is None and self._pipeline.device.type == "cuda"
                   and os.environ.get("OOB_DP_OVERLAP", "1") == "1"
                   and any(self._dp_engine._groups_of(l) is not None or l.sharded
                           for l in ex._layers))
        ex.grad_ready_hook = self._dp_engine.layer_ready if overlap else None

    def distribute_microbatches(self, templates: list[PipelineTemplate], global_num_microbatch: int) -> list[int]:
        """Integer stand-in for ``PipelineInstantiator._distribute_batch`` (instantiator.py:254-329, pyomo MINLP,
        control plane): proportional to each pipeline's GPU count, remainder to the largest pipelines first."""
        sizes = [t._num_nodes * t._num_gpus_per_node for t in templates]
        total = sum(sizes)
        out = [global_num_microbatch * s // total for s in sizes]
        order = sorted(range(len(sizes)), key=lambda i: (-sizes[i], i))
        for i in range(global_num_microbatch - sum(out)):
            out[order[i % len(order)]] += 1
        return out

    def make_pipeline(self, pipeline_id, template, ranks, dataloader, step) -> OobleckPipeline:
        return OobleckPipeline(pipeline_id=pipeline_id, pipeline_template=template, ranks=ranks, dataloader=dataloader,
                               step=step, training_args=self._hf_training_args, layer_cls=self._layer_cls,
                               transport_cls=self._transport_cls, nsplit=self._nsplit)

    def choose_plan(self) -> list[PipelineTemplate]:
        """Largest template that divides the world evenly, replicated (every BASELINE config has this shape)."""
        world_nodes = self._world_size // self._num_gpus_per_node
        for t in sorted(self._pipeline_templates, key=lambda t: -t._num_nodes):
            if world_nodes % t._num_nodes == 0:
                return [t] * (world_nodes // t._num_nodes)
        raise RuntimeError("no pipeline template fits the world size")

    def instantiate_pipelines(self, global_num_microbatch: int, plan: list[PipelineTemplate] | None = None):
        """engine.py:600-643."""
        if (not self._templates_injected and plan is None and self._layer_cls is None and torch.cuda.is_available()
                and os.environ.get("OOB_MEASURED_BALANCE", "1") == "1" and self._num_nodes > 1):
            from ..planning.profiler import measured_layer_results
            results = measured_layer_results(self._model, self._args.job.microbatch_size)
            self.layer_costs = [r._forward + r._backward for r in results.get()]
            self.layer_costs_source = "measured (CUDA events, fwd + bwd ms per layer kind, rank 0, broadcast)"
            if os.environ.get("OOB_TEMPLATE_SOURCE", "planner") == "planner":
                # the reference's flow (engine.py:453-500): profile -> PipelineTemplateGenerator.create_pipeline_templates
                from ..planning.pipeline_template import PipelineTemplateGenerator
                device_memory = torch.cuda.get_device_properties(torch.cuda.current_device()).total_memory
                lo, hi = node_range(results, self._num_nodes, self._num_gpus_per_node, device_memory)   # :490-512
                self.min_num_nodes = lo
                self._pipeline_templates = PipelineTemplateGenerator().create_pipeline_templates(
                    results, (lo, min(hi, len(self.layer_costs))), self._num_gpus_per_node)
                self.layer_costs_source += " -> template search (csrc/planning/template_search.cpp)"
            else:
                self._pipeline_templates = [balanced_template(self.layer_costs, n, self._num_gpus_per_node)
                                            for n in range(1, self._num_nodes + 1) if n <= len(self.layer_costs)]
                self.layer_costs_source += " -> min-max contiguous partition"
        plan = plan or self.choose_plan()
        num_microbatches = self.distribute_microbatches(plan, global_num_microbatch)
        ranks_list, used = [], 0
        for t in plan:
            n = t._num_nodes * t._num_gpus_per_node
            ranks_list.append(list(range(used, used + n)))
            used += n
        my_index = next(i for i, ranks in enumerate(ranks_list) if self._rank in ranks)
        dataloader = OobleckDataLoader(self._hf_training_args, self._dataset, LoaderType.Training, my_index,
                                       num_microbatches, 0, 0, device_resident=self._device_resident)
        pipelines = []
        self._pipeline = None
        for pid, (t, ranks) in enumerate(zip(plan, ranks_list)):     # every rank builds every pipeline (:118-149)
            p = self.make_pipeline(pid, t, ranks, dataloader, 0)
            pipelines.append(p)
            if p.my_pipeline:
                self._pipeline = p
        for p in pipelines:
            p.initialize_distributed_fsdp()
            p.initialize_distributed_pipeline()
        self._pipeline.initialize_execution(self._model)
        assert self._pipeline.communication is not None and self._pipeline.execution is not None
        self._dp_engine = DataParallelEngine(self, pipelines)
        self._install_dp_overlap()
        self._reconfiguration = ReconfigurationEngine(self, pipelines)
        self._step_aborted = False
        self._make_job_group()
        self._shadow = PeerShadow(self, self._pipeline) if self._peer_shadow and dist.is_initialized() else None
        if self._shadow is not None:
            self._shadow.refresh()          # step-0 state: a rank may be lost before the first optimizer step

    # -- training ----------------------------------------------------------------------------------------------------
    def _train_step(self):
        """engine.py:645-649."""
        self._pipeline.train()
        self._dp_engine.do_allreduce()
        self._pipeline.execution.optimizer_step()
        if self._shadow is not None:
            self._shadow.refresh()

    def _guarded_train_step(self) -> bool:
        """One ``_train_step`` that survives the loss of a peer (elastic runs: an agent pipe exists).

            1. unless a loss notification is already pending: run the pipeline's micro-batches, then drain the device;
               a wait on a neighbour that gave up (``transport.aborted()``: the peer is lost, or dropped the step) or a
               torch.distributed error marks the attempt as failed instead of propagating;
            2. vote: ONE MIN all-reduce of that flag over every rank of the job (``_job_group``).  The step goes on
               only if every rank finished its micro-batches and nobody has a notification pending; a dead rank makes
               the vote itself fail for everybody (gloo: peer reset; NCCL: released by the listener's abort);
            3. gradient exchange (all-reduce across replicas), then a SECOND vote on "my exchange completed": either
               all surviving ranks apply the optimizer step or none does (two-phase commit; the optimizer step itself
               is local), then the peer-shadow refresh;
               dropped  : gradients are zeroed, the queued reconfiguration is applied (waiting for the agent's message
               if the failure was noticed first), and the caller runs the step again on the new pipelines.

        Parameters are only written by ``optimizer_step``, the last action of a committed step, so a dropped step leaves
        the model exactly as the previous step left it.  Returns False for a dropped step."""
        if self._agent_pipe is None:
            self._train_step()
            return True
        on_gpu = torch.cuda.is_available() and self._pipeline.device.type == "cuda"
        failure: Exception | None = None
        ok = not self._notified
        global_step = self._pipeline._global_step
        if ok:
            try:
                self._pipeline.train()
                if on_gpu:
                    torch.cuda.synchronize()      # every wait of this step has either seen its data or given up
                if self._pipeline.communication.transport.aborted():
                    raise PipelineAborted("an inter-stage transfer was abandoned")
            except (PipelineAborted, RuntimeError) as e:
                ok, failure = False, e
        _dbg(f"step: pipeline ok={ok} failure={type(failure).__name__ if failure else None}; voting")
        try:
            agreed = self._vote(ok)
        except (PipelineAborted, RuntimeError) as e:
            _dbg(f"step: vote failed: {str(e)[:120]}")
            agreed = False
        _dbg(f"step: agreed={agreed}")
        if agreed:
            # second phase: gradients are exchanged (cross-replica all-reduce; a sharded stage's reduce-scatter), then a
            # second vote decides whether anybody applies them.  A rank that dies during the exchange fails the
            # collectives of its partners only -- without this vote those would drop the step while everybody else
            # commits it.  After a passed second vote the optimizer step is local: nothing can split the job any more.
            exchanged = True
            try:
                self._dp_engine.do_allreduce()
                for layer in self._pipeline.execution._layers:
                    layer.prepare_gradient_for_optim()
                if on_gpu:
                    torch.cuda.synchronize()
                if self._dp_engine.touches(self._lost_ranks):
                    raise PipelineAborted("a gradient all-reduce ran into a lost rank")   # never apply its output
            except (PipelineAborted, RuntimeError) as e:
                exchanged, failure = False, e
            try:
                agreed = self._vote(exchanged)
            except (PipelineAborted, RuntimeError) as e:
                _dbg(f"step: second vote failed: {str(e)[:120]}")
                agreed = False
            _dbg(f"step: gradients exchanged={exchanged} commit={agreed}")
            if agreed:
                self._pipeline.execution.optimizer_step()
        if agreed:
            if self._shadow is not None:
                self._shadow.refresh()      # a neighbour that dies in here leaves its mirror at the previous step
            return True
        self._pipeline._global_step = global_step      # the dropped step never happened
        try:
            self._pipeline.execution._optimizer.zero_grad()
            if on_gpu:
                torch.cuda.synchronize()
        except RuntimeError:
            pass                      # a poisoned stream: everything on it is rebuilt below anyway
        if not self._reconfiguration.poll() and not self._wait_for_notification():
            raise failure if failure is not None else PipelineAborted("step dropped but no loss was announced")
        return False

    # -- evaluation --------------------------------------------------------------------------------------------------
    def evaluate(self, num_microbatches: int | None = None) -> dict:
        """Validation loss of the current parameters: a forward-only pass of every pipeline over the first
        ``num_microbatches`` micro-batches of ``per_device_eval_batch_size`` sequences of the validation split (default:
        as many as the split holds), split between the pipelines like training micro-batches
        (``distribute_microbatches``).  The head computes the loss without writing logits (``oob_head_eval``).

        Returns, identically on every rank, ``loss`` (mean of the per-micro-batch mean losses, as HF's evaluation loop
        reports it), ``perplexity`` = exp(loss) (HF ``run_clm``), ``tokens`` (targets counted) and ``microbatches``.
        Training is not affected: parameters, gradients, moments, ``total_loss``, the step count, the LR schedule and
        the training data position stay as they were.  Every call starts at the beginning of the validation split."""
        mb = self._hf_training_args.per_device_eval_batch_size
        pipelines = self._reconfiguration._pipelines
        plan = [p._template for p in pipelines]
        # checked on every rank before any transfer: a first stage that ran out of data would leave the stages after
        # it waiting in a receive
        available = len(self._dataset.dataset["validation"]) // mb
        if num_microbatches is None:
            num_microbatches = available
        if not 1 <= num_microbatches <= available:
            raise ValueError(f"evaluate(): {num_microbatches} micro-batches of {mb} sequences asked for, the validation "
                             f"split holds {available}")
        counts = self.distribute_microbatches(plan, num_microbatches)
        my_index = next(i for i, p in enumerate(pipelines) if p is self._pipeline)
        loader = OobleckDataLoader(self._hf_training_args, self._dataset, LoaderType.Evaluation, my_index, counts, 0, 0,
                                   shuffle=False, device_resident=self._device_resident)
        res = self._pipeline.evaluate(self._model, loader, counts[my_index], mb)
        total = torch.zeros(3, dtype=torch.float64)
        if res is not None and self._pipeline.execution._shard_id == 0:   # one rank per pipeline reports
            total[0], total[1], total[2] = res[0], counts[my_index], res[1]
        group = self._eval_group()
        if group is not False:
            device = self._pipeline.device
            t = total.to(device)
            dist.all_reduce(t, group=group)
            total = t.cpu()
        loss = float(total[0]) / float(total[1])
        return {"loss": loss, "perplexity": math.exp(loss), "tokens": int(total[2]), "microbatches": int(total[1])}

    def _eval_group(self):
        """Communicator over every rank of the current pipelines: None = the world, False = this rank alone."""
        if not dist.is_initialized():
            return False
        ranks = sorted(r for p in self._reconfiguration._pipelines for r in p._ranks)
        if len(ranks) <= 1:
            return False
        if not self._reconfigured and len(ranks) == dist.get_world_size():
            return None
        return _communicator(ranks, self._comm_timeout)

    def _make_job_group(self):
        """Elastic runs: the communicator of the per-step vote -- every rank that currently trains."""
        self._job_ranks = sorted(r for p in self._reconfiguration._pipelines for r in p._ranks)
        self._job_group = None
        if self._agent_pipe is None or not dist.is_initialized() or len(self._job_ranks) <= 1:
            return
        self._job_group = _communicator(self._job_ranks, self._comm_timeout)

    def _vote(self, ok: bool) -> bool:
        if self._job_group is None:
            return ok
        device = self._pipeline.device
        flag = torch.tensor([1 if ok else 0], dtype=torch.int32, device=device)
        if device.type == "cpu":
            # gloo cannot abort a collective: once the listener has announced a loss this rank stops waiting for partners
            # that left the vote (NCCL: the listener aborts the communicator instead)
            run_interruptible(lambda: dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=self._job_group),
                              lambda: self._notified)
        else:
            dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=self._job_group)
        agreed = bool(flag.item())
        # an all-reduce released by ncclCommAbort leaves garbage behind: a communicator that turned out to contain a
        # lost rank while we were waiting cannot have produced a vote
        if self._lost_ranks & set(self._job_ranks):
            return False
        return agreed

    def _wait_for_notification(self, timeout: float = 60.0) -> bool:
        """A failure was noticed before the agent's lost-node message arrived: wait for the listener to queue it, then
        apply it."""
        t0 = time.perf_counter()
        while time.perf_counter() - t0 < timeout:
            if self._reconfiguration.poll():
                return True
            time.sleep(0.002)
        return False

    def train(self):
        assert self._hf_training_args.max_steps > 0
        done = 0
        while done < self._hf_training_args.max_steps:
            try:
                t0 = time.perf_counter()
                if self._guarded_train_step():
                    if self._agent_pipe is not None and torch.cuda.is_available() and \
                            self._pipeline.device.type == "cuda":
                        torch.cuda.synchronize()      # elastic runs: a step counts when its kernels have finished
                    self.step_end_times.append(time.perf_counter())
                    self.step_seconds.append(self.step_end_times[-1] - t0)
                    done += 1
            except StopIteration:
                self._pipeline.reset_iterator()                      # engine.py:660-663
                done += 1
        self.barrier()
        if torch.cuda.is_available():
            torch.cuda.synchronize()

    def barrier(self):
        """End-of-training rendezvous.  The world group still contains every rank that was ever lost (it is never
        rebuilt), so after a reconfiguration the barrier runs over a communicator of the survivors only."""
        if not dist.is_initialized():
            return
        if not self._reconfigured:
            dist.barrier()
            return
        alive = sorted(r for ranks in self._rank_map.values() for r in ranks) if self._rank_map else \
            sorted(r for p in self._reconfiguration._pipelines for r in p._ranks)
        if len(alive) <= 1:
            return
        dist.barrier(group=_communicator(alive, self._comm_timeout))
