"""Checker-side stage layer: the oracle's torch modules behind the ``Layer`` interface, so that the pipeline host logic
(schedule interpreter, wire protocol, DP groups, reconfiguration) can run on CPU with gloo -- in the tests, and as the
CPU arm of bench.py (``--impl reference``: P gloo processes running a real 1F1B step over these layers, BASELINE.md
section 4).  Test infrastructure like everything under oracle/: never imported by the product package."""
from __future__ import annotations

import torch

from oobleck_b200.execution.layer import HiddenGrad
from oobleck_b200.execution.optimizer import WarmupLR
from oobleck_b200.execution.sharding import ShardedFlatState, shard_param
from oracle import gpt2 as og
from oracle import optim as oo


class _Handle:
    def __init__(self, flat, process_group=None, sharded=False):
        self.flat_param = flat
        self.process_group = process_group
        self._sharding_strategy = "FULL_SHARD" if sharded else "NO_SHARD"

    @property
    def world_size(self) -> int:
        return self.process_group.size() if hasattr(self.process_group, "size") else 1


class OracleAdamW:
    def __init__(self, layers, lr, betas, eps, weight_decay=0.01):
        self.layers = list(layers)
        self.param_groups = [{"lr": lr, "betas": betas, "eps": eps, "weight_decay": weight_decay}]
        self.state = {}
        self._step = 0

    def step(self):
        self._step += 1
        g = self.param_groups[0]
        for l in self.layers:
            l.prepare_gradient_for_optim()
            l.opt_step += 1
            oo.adamw_step_(l.flat_param, l.flat_param.grad, l.exp_avg, l.exp_avg_sq, l.opt_step, g["lr"], g["betas"][0],
                           g["betas"][1], g["eps"], g["weight_decay"])
            l.refresh_planes()

    def zero_grad(self):
        for l in self.layers:
            l.zero_grad()


class OracleLayer:
    device_type = "cpu"

    @staticmethod
    def optimizer_factory():
        return OracleAdamW, WarmupLR

    fast_init = False      # bench.py's CPU arm: constant weights (timing does not depend on the values; drawing 1.5 G
                           # normal deviates on the host costs more than the sample itself)

    # Re-read the torch module's weights from ``flat_param`` before the first forward of every step.  For callers that write ``flat_param``
    # behind the layer's back and never say so -- the reference's own ``_copy_model_states`` broadcasts straight into it
    # (engine.py:284-306), which works there because FSDP's module parameters are views of the flat parameter.  Off by
    # default: bench.py's CPU arm would copy 6 GB per GPT-2-XL micro-batch for nothing.
    reload_every_forward = False

    def __init__(self, layer_id, spec, process_group=None, pre_stream=None, post_stream=None, *, microbatch_size,
                 num_pipe_buffers, workspace=None, nsplit=3, columns=1):
        self.layer_id = layer_id
        spec = getattr(spec, "spec", spec)
        self.spec = spec
        self.num_pipe_buffers = num_pipe_buffers
        d = og.GPT2Dims(n_embd=spec.n_embd, n_head=spec.n_head, n_layer=spec.n_layer, n_positions=spec.n_positions,
                        vocab_size=spec.vocab_size, layer_norm_epsilon=spec.layer_norm_epsilon)
        self.module = {"embed": og.EmbeddingLayer, "block": og.BlockLayer, "head": og.HeadLayer}[spec.kind](d)
        flat = torch.full((spec.num_params,), 0.01) if self.fast_init else spec.init_flat()
        k = process_group.size() if hasattr(process_group, "size") else 1
        self._group_size = k
        st = self._state = ShardedFlatState(spec.num_params, process_group, max(columns, k), "cpu")
        st.install_full_(flat)
        og.load_flat_(self.module, st.compute_param)
        self._param_handle = _Handle(st.param_shard, process_group, st.sharded)
        self.exp_avg, self.exp_avg_sq = st.exp_avg, st.exp_avg_sq
        self.saved = [None] * num_pipe_buffers
        self.opt_step = 0
        self._grads_final = False     # this step's gradient went through a collective: the module's copy is outdated

    @classmethod
    def create_layer_from_layer(cls, existing, pg, num_pipe_buffers=None):
        if num_pipe_buffers is not None and num_pipe_buffers > existing.num_pipe_buffers:
            existing.saved += [None] * (num_pipe_buffers - existing.num_pipe_buffers)
            existing.num_pipe_buffers = num_pipe_buffers
        return existing

    def state_tensors(self):
        return [self.flat_param, self.exp_avg, self.exp_avg_sq]

    @property
    def flat_param(self):
        return self._param_handle.flat_param

    @property
    def flat_grad(self):
        self.sync_grads()
        return self._param_handle.flat_param.grad

    @property
    def sharded(self):
        return self._state.sharded

    @property
    def full_param(self):
        return self._state.compute_param

    @property
    def full_grad(self):
        self.sync_grads()
        return self._state.compute_grad

    def sync_grads(self):
        """autograd accumulates in the module; the flat vector follows until a collective has rewritten it"""
        if not self._grads_final:
            self._state.compute_grad.copy_(og.flat_grads(self.module))

    def zero_grad(self):
        self.module.zero_grad()
        self._state.zero_grad()
        self._grads_final = False

    def load_flat_(self, flat):
        self._state.install_full_(flat)
        og.load_flat_(self.module, self._state.compute_param)

    def refresh_planes(self):
        if self._state.sharded:
            self._state.stale = True
        else:
            og.load_flat_(self.module, self._state.compute_param)

    def unshard_params(self, state=None):
        if self._state.unshard():
            og.load_flat_(self.module, self._state.compute_param)

    def reshard_params(self):
        pass

    def prepare_gradient_for_optim(self):
        self.sync_grads()
        if self._state.sharded:
            self._state.scatter_grads()
            self._grads_final = True

    def _shard_param(self, tensor, number):
        return shard_param(tensor, number)

    def remove_tensors(self):
        pass

    def __call__(self, inputs, buffer_id=0, total_loss=None):
        self.unshard_params()
        if self.reload_every_forward and not self._state.sharded and all(x is None for x in self.saved):
            # no micro-batch in flight (the first forward of a step): autograd holds no reference to the weights
            og.load_flat_(self.module, self._state.compute_param)
        ins = tuple(t.detach().requires_grad_(t.is_floating_point()) for t in inputs)
        outs = self.module(*ins)
        self.saved[buffer_id] = (ins, outs)
        if self.spec.kind == "head":
            if total_loss is not None:
                total_loss += outs[0].detach()
            return outs[0].detach(), outs[1].detach()
        return tuple(o.detach().requires_grad_(o.is_floating_point()) for o in outs)

    def backward(self, buffer_id, grad):
        ins, outs = self.saved[buffer_id]
        if self.spec.kind == "head":
            outs[0].backward()
        else:
            torch.autograd.backward(outs[0], grad.grad.view_as(outs[0]))
        self.saved[buffer_id] = None
        x = ins[0]
        return HiddenGrad(x.grad) if x.is_floating_point() else None

    def reduce_gradients(self, process_groups):
        self.prepare_gradient_for_optim()
        for chunk, pg in self._state.dp_chunks(process_groups):
            torch.distributed.all_reduce(chunk, group=getattr(pg, "group", pg))
        self._grads_final = True
