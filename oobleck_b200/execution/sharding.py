"""Intra-stage sharding of a stage layer's flat state (SURVEY 8(f3); oobleck/execution/layer.py:96-225, 262-291).

The reference wraps each layer in an FSDP ``FlatParamHandle`` with ``FULL_SHARD`` when the stage owns more than one GPU
(layer.py:100-102): every rank of the stage keeps ``1/k`` of the flat parameter, all-gathers it before every forward and
again before every backward of every micro-batch (pre_forward_hook / pre_backward_hook, :148-165), reduce-scatters the
gradient after every micro-batch backward into ``_saved_grad_shard`` (:167-225) and lets the optimizer work on the
shard.  Cross-replica all-reduce then runs per ``fsdp_index`` on the shards (:272-291), a layer that is NOT sharded in one
pipeline splitting its gradient with ``_shard_param`` (:262-270) to meet the shards of a pipeline where it is.

Same state ownership here, scheduled for the GPU:

* parameters change once per step, and HBM holds every gathered layer of a stage: the all-gather runs ONCE per
  step (lazily, before the first forward after ``optimizer_step``), in place -- the local shard is a view into the
  gathered buffer, so neither the gather nor the optimizer copies anything.  ``reshard_params`` therefore has nothing to
  free (2 x micro_batches all-gathers per layer and step in the reference, 1 here);
* gradients accumulate locally over all micro-batches in the full-size buffer the kernels write anyway, and ONE
  reduce-scatter per layer and step (SUM, like the reference: never averaged) produces the gradient shard -- started on
  the communication stream as soon as the layer's last micro-batch backward has retired when the overlap hook is
  installed (``DataParallelEngine.layer_ready``), otherwise right before the cross-replica reduction / optimizer;
* AdamW moments exist for the shard only.

Shard boundaries.  FSDP chunks the flat vector into ``ceil(n / k)`` pieces (``torch.chunk``) and zero-pads the last one.
The fused AdamW kernel works on 16-byte vectors and pipelines of different stage widths must agree on the boundaries of
what they all-reduce, so the unit here is ``round_up(ceil(n / columns), 8)`` elements, ``columns`` = number of shard
columns of the rank grid (``num_gpus_per_node``); a layer held by ``k`` ranks owns ``columns / k`` consecutive units per
rank.  For every GPT-2 stage layer and power-of-two ``k`` this coincides with FSDP's chunking (``n`` is a multiple of
``8 k``); ``shard_param`` below is the reference's ``_shard_param`` itself.

Device-agnostic on purpose (torch tensors + torch.distributed only): ``Layer`` (CUDA kernels) and the checker-side
``OracleLayer`` (gloo, CPU) share it, so the host logic is exercised by the CPU suite.
"""
from __future__ import annotations

import torch
import torch.distributed as dist


def shard_param(tensor: torch.Tensor, number: int) -> list[torch.Tensor]:
    """``Layer._shard_param`` of the reference (layer.py:262-270): ``number`` chunks of the flattened tensor, missing
    chunks zero-filled, the last one zero-padded to the size of the first."""
    chunks = list(torch.flatten(tensor).chunk(number))
    if len(chunks) < number:
        chunks = chunks + [torch.zeros_like(chunks[0]) for _ in range(number - len(chunks))]
    pad = chunks[0].numel() - chunks[-1].numel()
    if pad > 0:
        chunks[-1] = torch.nn.functional.pad(chunks[-1], [0, pad])
    return chunks


def shard_unit(numel: int, columns: int) -> int:
    """Elements per shard column (see the module docstring)."""
    per = -(-numel // columns)
    return (per + 7) // 8 * 8


class ShardedFlatState:
    """Flat parameter / gradient / moment storage of one layer.

    ``columns == 1`` is the reference's NO_SHARD branch and allocates exactly ``numel`` elements, nothing else.
    Otherwise ``full_param`` / ``full_grad`` hold ``columns * unit`` elements (zero tail), the compute kernels use their
    first ``numel`` elements, and rank ``index`` of the ``k`` holders owns elements ``[lo, hi)``."""

    def __init__(self, numel: int, group, columns: int, device):
        self.numel = numel
        self.columns = max(1, int(columns))
        self.k = group.size() if hasattr(group, "size") else 1
        self.index = max(0, group.rank_index()) if hasattr(group, "rank_index") else 0
        self.comm = getattr(group, "group", None)
        if self.columns % self.k:
            raise ValueError(f"a stage of {self.k} GPUs cannot hold {self.columns} shard columns evenly "
                             "(pipeline_template.h:57-84 repeats each stage rank columns / k times)")
        if self.k > 1 and self.comm is None:
            raise RuntimeError("a sharded layer needs the communicator of its stage (initialize_distributed_fsdp)")
        f32 = dict(dtype=torch.float32, device=device)
        if self.columns == 1:
            self.unit, self.padded = numel, numel
        else:
            self.unit = shard_unit(numel, self.columns)
            self.padded = self.unit * self.columns
        self.per_rank = self.padded // self.k                 # elements this rank owns
        self.lo, self.hi = self.index * self.per_rank, (self.index + 1) * self.per_rank
        self.full_param = torch.zeros(self.padded, **f32)
        self.full_grad = torch.zeros(self.padded, **f32)
        if self.k > 1:
            self.param_shard = self.full_param[self.lo:self.hi]            # a view: gather and optimizer work in place
            self.grad_shard = torch.zeros(self.per_rank, **f32)           # reduce-scatter output
            self.reduce_buffer = self.grad_shard
        else:   # the whole vector lives here; the zero tail only exists so that column slices have equal sizes
            self.param_shard = self.full_param if self.padded == numel else self.full_param[:numel]
            self.grad_shard = self.full_grad if self.padded == numel else self.full_grad[:numel]
            self.reduce_buffer = self.full_grad
        self.param_shard.grad = self.grad_shard
        self.exp_avg = torch.zeros(self.param_shard.numel(), **f32)
        self.exp_avg_sq = torch.zeros(self.param_shard.numel(), **f32)
        self.stale = False            # other ranks' shards in full_param are out of date
        self.grads_scattered = False  # grad_shard holds this step's reduce-scattered gradient
        self.gathers = 0              # collectives issued (tests / profiling)
        self.scatters = 0

    # the vectors the compute path reads and writes
    @property
    def compute_param(self) -> torch.Tensor:
        return self.full_param[:self.numel]

    @property
    def compute_grad(self) -> torch.Tensor:
        return self.full_grad[:self.numel]

    @property
    def sharded(self) -> bool:
        return self.k > 1

    def install_full_(self, flat: torch.Tensor) -> None:
        """Every holder has the whole vector (deterministic initial values, parity tests): nothing to gather."""
        self.full_param[:self.numel].copy_(flat.to(self.full_param.device, torch.float32))
        if self.padded > self.numel:
            self.full_param[self.numel:].zero_()
        self.stale = False

    def unshard(self) -> bool:
        """All-gather the shards into ``full_param`` if some are out of date.  Returns whether anything was fetched."""
        if not (self.sharded and self.stale):
            return False
        dist.all_gather_into_tensor(self.full_param, self.param_shard, group=self.comm)
        self.stale = False
        self.gathers += 1
        return True

    def scatter_grads(self, async_op: bool = False):
        """SUM reduce-scatter of the locally accumulated gradient over the stage's ranks (once per step)."""
        if not self.sharded or self.grads_scattered:
            return None
        self.grads_scattered = True
        self.scatters += 1
        return dist.reduce_scatter_tensor(self.grad_shard, self.full_grad, group=self.comm, async_op=async_op)

    def zero_grad(self) -> None:
        self.full_grad.zero_()
        if self.sharded:
            self.grad_shard.zero_()
        self.grads_scattered = False

    def dp_chunks(self, process_groups: dict) -> list[tuple[torch.Tensor, object]]:
        """Pair every cross-replica group this rank belongs to with the slice of its gradient that group reduces
        (layer.py:279-291).  Group ``fsdp_index`` covers column ``fsdp_index`` of the flat vector; consecutive columns
        that share a communicator are reduced in one call; single-member groups have nothing to do."""
        if self.columns == 1:
            assert len(process_groups) == 1, "one shard column but several cross-replica groups"
            pg = next(iter(process_groups.values()))
            return [(self.reduce_buffer, pg)] if pg.size() > 1 else []
        first_column = self.lo // self.unit if self.sharded else 0
        mine = self.per_rank // self.unit
        out: list[tuple[int, int, object]] = []
        for fsdp_index, pg in sorted(process_groups.items()):
            col = fsdp_index - first_column
            assert 0 <= col < mine, (f"cross-replica group of column {fsdp_index} on a rank that owns columns "
                                     f"{first_column}..{first_column + mine - 1}")
            if pg.size() <= 1:
                continue
            if out and out[-1][1] == col and getattr(out[-1][2], "group", out[-1][2]) is getattr(pg, "group", pg):
                out[-1] = (out[-1][0], col + 1, pg)
            else:
                out.append((col, col + 1, pg))
        return [(self.reduce_buffer[a * self.unit: b * self.unit], pg) for a, b, pg in out]
