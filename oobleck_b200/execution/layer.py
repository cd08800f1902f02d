"""``Layer``: one stage layer materialised on a GPU.

Replaces oobleck/execution/layer.py:40-291.  The reference wraps a deep-copied fx GraphModule in an FSDP
``FlatParamHandle`` and lets torch.autograd run it; here a layer is

* one flat fp32 parameter vector in HF ``parameters()`` order (``_param_handle.flat_param`` keeps the reference's
  attribute path so the reconfiguration / DP code that pokes it keeps working, engine.py:284-306),
* its flat fp32 gradient (``flat_param.grad``), AdamW moments and the split-bf16 planes the wgmma GEMMs read,
* per pipe-buffer activation contexts that the hand-written forward fills and the hand-written backward consumes
  (no autograd graph, no checkpoint recompute -- layer.py:93-94 re-runs every block forward in backward).

A stage that owns several GPUs shards this state across them (layer.py:96-142, 167-225 -- FSDP ``FULL_SHARD``): see
``sharding.py`` for the GPU schedule of it (one in-place all-gather and one reduce-scatter per layer and STEP).  Every
BASELINE config runs one GPU per stage, the reference's ``NO_SHARD`` branch (layer.py:100-102), which allocates exactly
what it did before sharding existed.
"""
from __future__ import annotations

import ctypes as C
import math
import os
from dataclasses import dataclass

import torch

from .. import lib as L
from ..module.model import StageLayerSpec
from .sharding import ShardedFlatState, shard_param


from ..lib import OobBlockCtx, OobBwdScratch, OobDims, OobHeadCtx, OobLayerParams  # noqa: E402


# default numerics of the backward GEMMs (see Layer.__init__); bench.py / tests flip it explicitly.  On: measured
# +25 % tokens/s on GPT-2-XL with unchanged gradient parity (worst 3.3e-6 of max vs 2.4e-6, tests/test_stage_gpu.py)
DEFAULT_BWD_FP16 = os.environ.get("OOB_BWD_FP16", "1") == "1"


def _stream() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _round8(n: int) -> int:
    return (n + 7) // 8 * 8


def alloc_block_ctx(batch: int, seq: int, n_embd: int, n_head: int, nplanes: int,
                    device: torch.device) -> tuple[dict, OobBlockCtx]:
    """The activations one block forward saves (``oob_block_ctx``) for ``batch`` sequences: the tensors and the struct
    of their addresses.  ``nplanes`` planes for every buffer a forward GEMM and a wgrad read."""
    M, E = batch * seq, n_embd
    f32 = dict(dtype=torch.float32, device=device)
    bf = dict(dtype=torch.bfloat16, device=device)
    t = {"ln1_planes": torch.empty(nplanes, M, E, **bf), "ln1_mean": torch.empty(M, **f32),
         "ln1_rstd": torch.empty(M, **f32), "qkv_planes": torch.empty(3, M, 3 * E, **bf),
         "att": torch.empty(M, E, **f32), "att_planes": torch.empty(nplanes, M, E, **bf),
         "lse": torch.empty(batch * n_head * seq, **f32), "x2": torch.empty(M, E, **f32),
         "ln2_planes": torch.empty(nplanes, M, E, **bf), "ln2_mean": torch.empty(M, **f32),
         "ln2_rstd": torch.empty(M, **f32), "fc": torch.empty(M, 4 * E, **f32),
         "gelu_planes": torch.empty(nplanes, M, 4 * E, **bf)}
    return t, OobBlockCtx(**{k: v.data_ptr() for k, v in t.items()})


def init_tensors(layer, device) -> None:
    """oobleck/execution/layer.py:26-37 (called by planning/profiler.py:272-274 for every ``model.layers`` entry before
    profiling): put the layer's tensors on ``device``.  The reference fills parameters with ``torch.rand`` ("TODO: must
    use checkpointed data"); here the layer gets its deterministic HF-style initial values (``StageLayerSpec.init_flat``)
    when its kernels-side ``Layer`` is built, which happens on the first call (the micro-batch shape is not known
    before)."""
    device = torch.device(device)
    if device.type != "cuda":
        raise L.OobleckB200Error("oobleck_b200 stage layers live on CUDA devices only (there is no CPU path)")
    L.load()   # fail loudly if the CUDA extension is missing
    layer.to(device)


class StageWorkspace:
    """Backward temporaries of one stage (``oob_bwd_scratch``) plus the two ping-pong gradient buffers that carry
    d(hidden) from layer to layer.  Shared by all layers of the stage: backward is serial on one stream."""

    def __init__(self, microbatch: int, seq: int, n_embd: int, n_head: int, device: torch.device):
        M, E = microbatch * seq, n_embd
        f32 = dict(dtype=torch.float32, device=device)
        bf = dict(dtype=torch.bfloat16, device=device)
        lib = L.load()
        nparts = max(lib.oob_ln_bwd_partials_floats(E), lib.oob_colsum_partials_floats(4 * E))
        # Two scratch sets, alternated between consecutive layer backwards: the weight-gradient kernels of layer l run
        # on the library's side stream while the main stream is already in layer l-1 (oob_bwd_scratch.defer_join).
        self.sets, self.scratches = [], []
        for _ in range(2):
            t = {
                "dfc": torch.empty(M, 4 * E, **f32), "dfc_planes": torch.empty(3, M, 4 * E, **bf),
                "dln": torch.empty(M, E, **f32), "dx2": torch.empty(M, E, **f32),
                "dx2_planes": torch.empty(3, M, E, **bf),
                "datt": torch.empty(M, E, **f32), "datt_planes": torch.empty(3, M, E, **bf),
                "delta": torch.empty(microbatch * n_head * seq, **f32),
                "dqkv": torch.empty(M, 3 * E, **f32), "dqkv_planes": torch.empty(3, M, 3 * E, **bf),
                "partials": torch.empty(nparts, **f32),
                "partials_side": torch.empty(lib.oob_colsum_partials_floats(4 * E), **f32),
            }
            self.sets.append(t)
            self.scratches.append(OobBwdScratch(defer_join=1, **{k: v.data_ptr() for k, v in t.items()}))
        self.t, self.scratch = self.sets[0], self.scratches[0]
        self._scratch_flip = 0
        self.dx = [torch.empty(M, E, **f32) for _ in range(2)]
        self.dx_planes = [torch.empty(3, M, E, **bf) for _ in range(2)]
        self.recv_planes = torch.empty(3, M, E, **bf)  # planes of a gradient received from the next stage
        self.flip = 0

    def next_dx(self):
        self.flip ^= 1
        return self.dx[self.flip], self.dx_planes[self.flip]

    def next_scratch(self) -> OobBwdScratch:
        self._scratch_flip ^= 1
        return self.scratches[self._scratch_flip]

    def join(self) -> None:
        """Main stream waits for the side stream's weight-gradient kernels (end of a backward pass)."""
        L.call("oob_side_join", _stream())


class EvalWorkspace:
    """Forward-only temporaries of one stage at the evaluation micro-batch size (``Layer.evaluate``).  Nothing is saved
    for a backward, so ONE ``oob_block_ctx`` serves every block of the stage, two ping-pong buffers carry the hidden
    state from layer to layer, and the head needs ln_f's planes and the LM head's row partials, never logits.
    ``acc`` accumulates (sum of micro-batch mean losses, targets counted) on the device."""

    def __init__(self, microbatch: int, seq: int, n_embd: int, n_head: int, vocab: int, device: torch.device):
        self.mb, self.T = microbatch, seq
        M, E = microbatch * seq, n_embd
        self.device = device
        f32 = dict(dtype=torch.float32, device=device)
        self.hidden = [torch.empty(microbatch, seq, E, **f32) for _ in range(2)]
        self._n_embd, self._n_head, self._vocab = E, n_head, vocab
        self._ctx: dict[int, tuple] = {}      # plane count -> (tensors, oob_block_ctx)
        self._head: dict[int, dict] = {}      # ln_f plane count -> tensors
        self.acc = torch.zeros(2, dtype=torch.float64, device=device)

    def next_hidden(self, avoid: torch.Tensor | None = None) -> torch.Tensor:
        """A hidden buffer that is not ``avoid`` (the layer's input)."""
        a = avoid.data_ptr() if avoid is not None else None
        return self.hidden[1] if self.hidden[0].data_ptr() == a else self.hidden[0]

    def block_ctx(self, nplanes: int) -> OobBlockCtx:
        if nplanes not in self._ctx:
            self._ctx[nplanes] = alloc_block_ctx(self.mb, self.T, self._n_embd, self._n_head, nplanes, self.device)
        return self._ctx[nplanes][1]

    def head_buffers(self, nplanes: int) -> dict:
        if nplanes not in self._head:
            M, E = self.mb * self.T, self._n_embd
            f32 = dict(dtype=torch.float32, device=self.device)
            self._head[nplanes] = {
                "lnf_planes": torch.empty(nplanes, M, E, dtype=torch.bfloat16, device=self.device),
                "mean": torch.empty(M, **f32), "rstd": torch.empty(M, **f32),
                "partials": torch.empty(L.load().oob_head_eval_partials_floats(M, self._vocab), **f32),
                "row_loss": torch.empty(M, **f32), "loss": torch.zeros(1, **f32)}
        return self._head[nplanes]


@dataclass
class HiddenGrad:
    """Gradient w.r.t. a hidden state travelling backwards through a stage: fp32 + (optionally) its planes."""
    grad: torch.Tensor
    planes: torch.Tensor | None = None


class _ParamHandle:
    """Just enough of FSDP's FlatParamHandle for the callers that reach through ``layer._param_handle``."""

    def __init__(self, flat_param: torch.Tensor, process_group, sharded: bool = False):
        self.flat_param = flat_param
        self.process_group = process_group
        # layer.py:100-102: FULL_SHARD when the per-layer group has more than one rank
        self._sharding_strategy = "FULL_SHARD" if sharded else "NO_SHARD"

    @property
    def uses_sharded_strategy(self) -> bool:
        return self._sharding_strategy != "NO_SHARD"

    @property
    def world_size(self) -> int:
        """FlatParamHandle.world_size: ranks the layer's state is spread over (read by the reference's tests,
        tests/execution/test_engine.py:996)."""
        return self.process_group.size() if hasattr(self.process_group, "size") else 1


class Layer:
    """Constructor keeps the reference's positional order (layer.py:71-78)."""

    device_type = "cuda"
    supports_deferred_init = True     # accepts init_values=False (see __init__)

    @classmethod
    def make_workspace(cls, model, microbatch_size: int, device) -> "StageWorkspace":
        spec = model.layers[0]
        return StageWorkspace(microbatch_size, spec.n_positions, spec.n_embd, spec.n_head, torch.device(device))

    @classmethod
    def make_eval_workspace(cls, model, microbatch_size: int, device) -> "EvalWorkspace":
        spec = model.layers[0]
        return EvalWorkspace(microbatch_size, spec.n_positions, spec.n_embd, spec.n_head, spec.vocab_size,
                             torch.device(device))

    def __init__(self, layer_id: int, layer: StageLayerSpec, process_group=None, pre_stream=None, post_stream=None, *,
                 microbatch_size: int, num_pipe_buffers: int, workspace: StageWorkspace | None = None,
                 nsplit: int = 3, device: torch.device | None = None, seq_len: int | None = None,
                 bwd_fp16: bool | None = None, init_values: bool = True, columns: int = 1):
        L.load()  # fail loudly if the CUDA extension is missing
        if not torch.cuda.is_available():
            raise L.OobleckB200Error("oobleck_b200.Layer needs a CUDA device (there is no CPU path)")
        self.layer_id = layer_id
        self.spec = getattr(layer, "spec", layer)      # a model.layers entry (StageLayer) or the bare spec
        layer = self.spec
        self.device = device or torch.device("cuda", torch.cuda.current_device())
        self._rank_index = process_group.rank_index() if hasattr(process_group, "rank_index") else 0
        self._group_size = process_group.size() if hasattr(process_group, "size") else 1
        self.pre_stream, self.post_stream = pre_stream, post_stream
        self.nsplit = nsplit
        self.mb = microbatch_size
        self.T = seq_len or layer.n_positions
        self.num_pipe_buffers = num_pipe_buffers
        self.workspace = workspace

        n = layer.num_params
        self.numel = n
        self.plane_stride = _round8(n)
        # ``init_values=False``: the layer is built to RECEIVE its state (reconfiguration moves parameters and moments
        # into it); generating 30-80 M random numbers per layer on the host was most of the rebuild time
        st = self._state = ShardedFlatState(n, process_group, max(columns, self._group_size), self.device)
        if init_values:     # deterministic: every holder of a sharded layer starts from the same full vector
            st.install_full_(layer.init_flat())
        else:
            st.stale = st.sharded   # the shard arrives from another rank; the rest is gathered on first use
        self._param_handle = _ParamHandle(st.param_shard, process_group, st.sharded)
        self.exp_avg, self.exp_avg_sq = st.exp_avg, st.exp_avg_sq
        # forward GEMMs read fp16 x 2 planes (3 tensor-core products, fp32-grade for bounded-range operands); the
        # bf16 x 3 planes stay for the backward GEMMs: 5-plane buffers (include/oobleck_b200.h)
        self.fwd_fp16 = 1 if nsplit == 3 else 0
        # backward GEMMs on loss-scaled fp16 pairs as well (3 products); activation gradients inside the stage -- and
        # across stage boundaries, both sides are this engine -- are carried multiplied by ``loss_scale``
        tokens = max(1, microbatch_size * ((seq_len or layer.n_positions) - 1))
        self.loss_scale = float(16 * 2 ** int(math.floor(math.log2(tokens))))   # dlogits * loss_scale is O(16)
        # placed here because the plane layout depends on it: all-fp16 mode keeps pair-only buffers
        self.bwd_fp16 = 1 if (self.fwd_fp16 and (DEFAULT_BWD_FP16 if bwd_fp16 is None else bwd_fp16)) else 0
        # plane-set codes handed to the producers (include/oobleck_b200.h): ``nplanes`` for the weights and every saved
        # activation a GEMM reads, ``grad_code`` for activation gradients; ``nplane_count`` planes are allocated.  The
        # embedding layer feeds no GEMM (wte / wpe are gathered in fp32): it carries no planes at all.
        act_code = L.PLANES_FP16_PAIR if self.bwd_fp16 else (L.PLANES_BF16X3_FP16_PAIR if self.fwd_fp16 else 3)
        self.nplanes = 0 if layer.kind == "embed" else act_code
        self.nplane_count = L.planes_count(self.nplanes)
        self.grad_code = L.PLANES_FP16_PAIR if self.bwd_fp16 else 3
        self.planes = (torch.empty(self.nplane_count, self.plane_stride, dtype=torch.bfloat16, device=self.device)
                       if self.nplanes else None)
        # AdamW step count of THIS layer's moments: travels with exp_avg / exp_avg_sq through reconfigurations so the
        # bias correction matches the moments (optimizer.py)
        self.opt_step = 0
        if init_values:
            self._split_planes()

        self.dims = self._dims(self.mb)
        self._alloc_contexts()

    def _dims(self, batch: int) -> OobDims:
        """``oob_dims`` of this layer for micro-batches of ``batch`` sequences."""
        s, V = self.spec, self.spec.vocab_size
        return OobDims(batch, self.T, s.n_embd, s.n_head, V, (V + 63) // 64 * 64, s.layer_norm_epsilon, self.nsplit,
                       self.fwd_fp16, self.bwd_fp16, self.loss_scale)

    # -- parameters ------------------------------------------------------------------------------------------------
    @property
    def flat_param(self) -> torch.Tensor:
        return self._param_handle.flat_param

    @property
    def flat_grad(self) -> torch.Tensor:
        """Gradient of ``flat_param``: the whole vector, or -- sharded -- this rank's reduce-scattered shard."""
        return self._param_handle.flat_param.grad

    @property
    def sharded(self) -> bool:
        return self._state.sharded

    @property
    def full_param(self) -> torch.Tensor:
        """The ``numel`` parameters the kernels read (== ``flat_param`` unless the stage shards the layer)."""
        return self._state.compute_param

    @property
    def full_grad(self) -> torch.Tensor:
        """The ``numel`` gradients the kernels accumulate into, local to this rank."""
        return self._state.compute_grad

    def planes_ptr(self) -> int:
        return self.planes.data_ptr() if self.planes is not None and self.planes.numel() else 0

    def optimizer_planes_ptr(self) -> int:
        """Planes the fused AdamW refreshes while it writes the parameters: only when the whole vector is updated
        here.  A sharded layer splits its planes after the next all-gather instead (``unshard_params``)."""
        return 0 if self._state.sharded else self.planes_ptr()

    def _params_struct(self) -> OobLayerParams:
        return OobLayerParams(self._state.full_param.data_ptr(), self.planes_ptr(), self.plane_stride,
                              self._state.full_grad.data_ptr())

    def _split_planes(self) -> None:
        if not self.nplanes:
            return
        L.call("oob_split_planes", C.c_void_p(self._state.full_param.data_ptr()), C.c_void_p(self.planes.data_ptr()),
               self.numel, self.plane_stride, self.nplanes, _stream())

    def refresh_planes(self) -> None:
        """``flat_param`` was written from outside (a received state): make the copies the kernels read current.  A
        sharded layer only notes that its gathered copy is out of date; the gather itself is a collective and runs
        when every holder reaches its next forward."""
        if self._state.sharded:
            self._state.stale = True
            return
        self._split_planes()

    def load_flat_(self, flat: torch.Tensor) -> None:
        """Install explicit weights -- the WHOLE vector, on every holder (parity tests, reconfiguration copies)."""
        assert flat.numel() == self.numel
        self._state.install_full_(flat)
        self._split_planes()

    # -- sharding (layer.py:117-165) -----------------------------------------------------------------------------------
    def unshard_params(self, state=None) -> None:
        """layer.py:117-133.  Gathers only if the shards changed since the last gather (once per step); the reference
        gathers before every forward and every backward."""
        if self._state.unshard():
            self._split_planes()

    def reshard_params(self) -> None:
        """layer.py:135-144.  Nothing to free: the gathered copy stays resident until the optimizer invalidates it
        (sharding.py)."""

    def prepare_gradient_for_optim(self) -> None:
        """FSDP's name for "make ``flat_param.grad`` the gradient the optimizer consumes" (layer.py:276): for a sharded
        layer, the SUM reduce-scatter of the locally accumulated gradient, unless it already ran for this step."""
        self._state.scatter_grads()

    def _shard_param(self, tensor: torch.Tensor, number: int) -> list[torch.Tensor]:   # layer.py:262-270
        return shard_param(tensor, number)

    def state_tensors(self) -> list[torch.Tensor]:
        """What has to move when this layer changes owner: parameters and both Adam moments (the reference moves
        ``flat_param`` only, engine.py:284-306, and silently restarts the moments).  Sharded: this rank's shards."""
        return [self.flat_param, self.exp_avg, self.exp_avg_sq]

    def adopt_state_(self, other: "Layer") -> None:
        """Take over parameters, gradients-in-progress, moments and step count of ``other`` (same layer id, same
        device): used when a reused layer needs more pipe buffers than it was built with."""
        assert other.numel == self.numel and other.layer_id == self.layer_id
        assert other._state.padded == self._state.padded and other._state.k == self._state.k
        self._state.full_param.copy_(other._state.full_param)
        self._state.full_grad.copy_(other._state.full_grad)
        self.exp_avg.copy_(other.exp_avg)
        self.exp_avg_sq.copy_(other.exp_avg_sq)
        self._state.stale = other._state.stale
        self.opt_step = other.opt_step
        if not self._state.stale:
            self._split_planes()

    def grow_pipe_buffers(self, num_pipe_buffers: int) -> None:
        """Re-allocate the per-slot activation contexts for a deeper schedule; parameters and optimizer state are
        untouched (contexts only live inside a train step)."""
        if num_pipe_buffers > self.num_pipe_buffers:
            self.num_pipe_buffers = num_pipe_buffers
            self._alloc_contexts()

    def zero_grad(self) -> None:
        self._state.zero_grad()

    def remove_tensors(self) -> None:  # layer.py:66-69
        empty = torch.tensor([], device=self.device)
        if self.flat_param.grad is not None:
            self.flat_param.grad = None
        self.flat_param.data = empty
        st = self._state
        st.full_param = st.full_grad = st.grad_shard = st.reduce_buffer = st.exp_avg = st.exp_avg_sq = empty
        self.planes = self.exp_avg = self.exp_avg_sq = empty
        self.ctx_tensors, self.out = [], []

    @classmethod
    def create_layer_from_layer(cls, existing_layer: "Layer", process_group,
                                num_pipe_buffers: int | None = None) -> "Layer":  # layer.py:41-64
        if existing_layer._state.sharded or (hasattr(process_group, "size") and process_group.size() > 1):
            old = getattr(existing_layer._param_handle.process_group, "ranks", None)
            if old != getattr(process_group, "ranks", None):
                raise NotImplementedError(f"layer {existing_layer.layer_id}: re-sharding a live layer over a different "
                                          f"set of stage ranks ({old} -> {getattr(process_group, 'ranks', None)})")
        existing_layer._param_handle.process_group = process_group
        if num_pipe_buffers is not None:
            existing_layer.grow_pipe_buffers(num_pipe_buffers)   # never shrinks; weights / moments stay in place
        return existing_layer

    # -- activations -----------------------------------------------------------------------------------------------
    def _alloc_contexts(self) -> None:
        M, E, H = self.mb * self.T, self.spec.n_embd, self.spec.n_head
        f32 = dict(dtype=torch.float32, device=self.device)
        bf = dict(dtype=torch.bfloat16, device=self.device)
        self.ctx_tensors, self.ctx, self.out, self.saved_in = [], [], [], [None] * self.num_pipe_buffers
        for _ in range(self.num_pipe_buffers):
            if self.spec.kind == "block":
                t, ctx = alloc_block_ctx(self.mb, self.T, E, H, self.nplane_count, self.device)
                self.ctx.append(ctx)
                self.out.append(torch.empty(self.mb, self.T, E, **f32).requires_grad_(True))
            elif self.spec.kind == "head":
                Vp = self.dims.vocab_padded
                t = {"lnf_planes": torch.empty(self.nplane_count, M, E, **bf),
                     "mean": torch.empty(M, **f32),
                     "rstd": torch.empty(M, **f32), "logits": torch.empty(M, Vp, **f32),
                     "dlogits_planes": torch.empty(3, M, Vp, **bf), "row_loss": torch.empty(M, **f32),
                     "loss": torch.zeros(1, **f32)}
                self.ctx.append(OobHeadCtx(**{k: v.data_ptr() for k, v in t.items()}))
                self.out.append(t["loss"])
            else:
                t = {}
                self.ctx.append(None)
                self.out.append(torch.empty(self.mb, self.T, E, **f32).requires_grad_(True))
            self.ctx_tensors.append(t)

    # -- compute ---------------------------------------------------------------------------------------------------
    def __call__(self, inputs: tuple, buffer_id: int = 0, total_loss: torch.Tensor | None = None) -> tuple:
        return self.forward(inputs, buffer_id, total_loss)

    def forward(self, inputs: tuple, buffer_id: int = 0, total_loss: torch.Tensor | None = None) -> tuple:
        """tuple in, tuple out, like the fx shards (sharding.py:86-96)."""
        self.saved_in[buffer_id] = inputs
        if self._state.sharded:
            self.unshard_params()
        if self.spec.kind != "head":
            return self._forward_into(inputs, self.dims, self.out[buffer_id], self.ctx[buffer_id])
        hidden, labels = inputs
        assert hidden.dtype == torch.float32 and hidden.is_contiguous()
        assert labels.dtype == torch.int64 and labels.is_contiguous()
        p = self._params_struct()
        L.call("oob_head_forward", C.byref(self.dims), C.byref(p), C.c_void_p(hidden.data_ptr()),
               C.c_void_p(labels.data_ptr()), C.byref(self.ctx[buffer_id]),
               C.c_void_p(0 if total_loss is None else total_loss.data_ptr()), _stream())
        loss = self.ctx_tensors[buffer_id]["loss"][0]  # 0-dim view, like HF's scalar loss
        return loss, self.ctx_tensors[buffer_id]["logits"]

    def _forward_into(self, inputs: tuple, dims: OobDims, y: torch.Tensor, ctx: OobBlockCtx | None) -> tuple:
        """Embedding or block forward of ``dims.batch`` sequences into ``y``; a block saves its activations in
        ``ctx``.  Shared by training (``forward``) and evaluation (``evaluate``)."""
        M, E = dims.batch * dims.seq, dims.n_embd
        if self.spec.kind == "embed":
            input_ids, _attention_mask, labels = inputs
            assert input_ids.dtype == torch.int64 and input_ids.is_contiguous() and input_ids.numel() == M
            w = self._state.full_param
            L.call("oob_embedding_fwd", C.c_void_p(input_ids.data_ptr()), C.c_void_p(w.data_ptr()),
                   C.c_void_p(w.data_ptr() + self.spec.vocab_size * E * 4), C.c_void_p(y.data_ptr()), M, dims.seq, E,
                   _stream())
            return y, labels
        hidden, labels = inputs
        assert hidden.dtype == torch.float32 and hidden.is_contiguous() and hidden.numel() == M * E
        L.call("oob_block_forward", C.byref(dims), C.byref(self._params_struct()), C.c_void_p(hidden.data_ptr()),
               C.c_void_p(y.data_ptr()), C.byref(ctx), _stream())
        return y, labels

    def backward(self, buffer_id: int, grad: HiddenGrad | None) -> HiddenGrad | None:
        """Hand-written backward of this layer for the micro-batch held in ``buffer_id`` (layer.py:250-260 runs
        torch.autograd here).  Parameter gradients accumulate into ``flat_grad``."""
        kind = self.spec.kind
        inputs = self.saved_in[buffer_id]
        ws = self.workspace
        if self._state.sharded:
            self.unshard_params()     # pre_backward_hook (layer.py:159-165); a no-op unless the shards changed
        p = self._params_struct()
        if kind == "head":
            hidden = inputs[0]
            dx, dxp = ws.next_dx()
            L.call("oob_head_backward", C.byref(self.dims), C.byref(p), C.c_void_p(hidden.data_ptr()),
                   C.byref(self.ctx[buffer_id]), C.byref(ws.next_scratch()), C.c_void_p(dx.data_ptr()),
                   C.c_void_p(dxp.data_ptr()), _stream())
            return HiddenGrad(dx, dxp)
        assert grad is not None
        E = self.spec.n_embd
        if kind == "block":
            hidden = inputs[0]
            if grad.planes is None:  # arrived from the next stage as fp32 only: split it here
                dy_planes = ws.recv_planes
                L.call("oob_split_planes", C.c_void_p(grad.grad.data_ptr()), C.c_void_p(dy_planes.data_ptr()),
                       grad.grad.numel(), dy_planes.stride(0), self.grad_code, _stream())
                grad = HiddenGrad(grad.grad, dy_planes)
            dx, dxp = ws.next_dx()
            if dx.data_ptr() == grad.grad.data_ptr():
                dx, dxp = ws.next_dx()
            L.call("oob_block_backward", C.byref(self.dims), C.byref(p), C.c_void_p(hidden.data_ptr()),
                   C.byref(self.ctx[buffer_id]), C.c_void_p(grad.grad.data_ptr()), C.c_void_p(grad.planes.data_ptr()),
                   C.byref(ws.next_scratch()), C.c_void_p(dx.data_ptr()), C.c_void_p(dxp.data_ptr()), _stream())
            return HiddenGrad(dx, dxp)
        # embedding
        input_ids = inputs[0]
        g = self._state.full_grad
        L.call("oob_embedding_bwd", C.c_void_p(input_ids.data_ptr()), C.c_void_p(grad.grad.data_ptr()),
               C.c_void_p(g.data_ptr()), C.c_void_p(g.data_ptr() + self.spec.vocab_size * E * 4), self.mb, self.T, E,
               (1.0 / self.loss_scale) if self.bwd_fp16 else 1.0, _stream())
        return None

    # -- evaluation ----------------------------------------------------------------------------------------------------
    def evaluate(self, inputs: tuple, eval_ws: EvalWorkspace) -> tuple:
        """Forward-only pass of this layer at the evaluation micro-batch size ``eval_ws.mb``: tuple in, tuple out like
        ``forward``.  Writes only ``eval_ws``: contexts, ``saved_in``, ``out``, gradients, moments and every loss of
        the training path are untouched.  The head returns ``(loss,)`` and adds into ``eval_ws.acc``."""
        kind = self.spec.kind
        if self._state.sharded:
            self.unshard_params()     # the same all-gather a forward runs (a no-op unless the shards changed)
        assert eval_ws.T == self.T      # the workspace's buffers are sized for the sequences the kernels write
        dims = self._dims(eval_ws.mb)
        if kind != "head":
            ctx = eval_ws.block_ctx(self.nplane_count) if kind == "block" else None
            return self._forward_into(inputs, dims, eval_ws.next_hidden(avoid=inputs[0]), ctx)
        hidden, labels = inputs
        assert hidden.dtype == torch.float32 and hidden.is_contiguous()
        assert hidden.numel() == dims.batch * dims.seq * dims.n_embd
        assert labels.dtype == torch.int64 and labels.is_contiguous()
        p = self._params_struct()
        # ln_f's planes feed only the LM-head GEMM: the fp16 pair when the forward reads pairs, else nsplit bf16 planes
        lnf_code = L.PLANES_FP16_PAIR if self.fwd_fp16 else self.nsplit
        t = eval_ws.head_buffers(L.planes_count(lnf_code))
        L.call("oob_head_eval", C.byref(dims), C.byref(p), C.c_void_p(hidden.data_ptr()),
               C.c_void_p(labels.data_ptr()), C.c_void_p(t["lnf_planes"].data_ptr()), lnf_code,
               C.c_void_p(t["mean"].data_ptr()), C.c_void_p(t["rstd"].data_ptr()),
               C.c_void_p(t["partials"].data_ptr()), C.c_void_p(t["row_loss"].data_ptr()),
               C.c_void_p(t["loss"].data_ptr()), C.c_void_p(eval_ws.acc.data_ptr()), _stream())
        return (t["loss"][0],)

    # -- data parallel -----------------------------------------------------------------------------------------------
    def reduce_gradients(self, process_groups: dict, async_op: bool = False):
        """layer.py:272-291: SUM all-reduce of the gradient over the cross-replica group(s); never averaged.  With one
        GPU per stage there is exactly one (fsdp_index -> group) entry and the whole flat gradient is reduced.  A
        sharded layer first reduce-scatters over its stage (once per step) and reduces its shard; a layer that shares
        shard columns with a sharded replica reduces column by column (``ShardedFlatState.dp_chunks``).  ``async_op``:
        return the NCCL work handles instead of waiting (the caller overlaps the reduction with the rest of the
        backward pass)."""
        works = []
        w = self._state.scatter_grads(async_op=async_op)
        if w is not None and async_op:
            w.wait()     # stream-side: the cross-replica reduction below (another communicator) reads the shard
        for chunk, pg in self._state.dp_chunks(process_groups):
            w = torch.distributed.all_reduce(chunk, group=getattr(pg, "group", pg), async_op=async_op)
            if async_op:
                works.append(w)
        return works
