"""Optimizer + LR schedule of a stage (oobleck/execution/pipeline.py:117-127, 241-244).

``FusedAdamW`` == ``torch.optim.AdamW(flat_params, lr, betas, eps, fused=True)`` with torch's default
weight_decay 0.01, one fused CUDA kernel per layer that also refreshes the split-bf16 planes the GEMMs read.
``WarmupLR`` == deepspeed ``WarmupLR(optimizer, <2nd positional>)``: the reference passes HF's warm-up step count
(0) as ``warmup_min_lr``; everything else is deepspeed's default (max 1e-3, 1000 steps, log warm-up).
"""
from __future__ import annotations

import ctypes as C
import math

import torch

from .. import lib as L


class FusedAdamW:
    def __init__(self, layers, lr: float = 5e-5, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 0.01):
        self.layers = list(layers)
        self.param_groups = [{"lr": lr, "betas": betas, "eps": eps, "weight_decay": weight_decay,
                              "params": [l.flat_param for l in self.layers]}]
        self._step = 0
        # torch-like state view: flat_param -> {"step", "exp_avg", "exp_avg_sq"} (test_layer.py:125-136)
        self.state = {}

    def step(self) -> None:
        self._step += 1
        g = self.param_groups[0]
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        for l in self.layers:
            # the bias correction follows the layer's own moments (torch keeps ``step`` per parameter too): a layer
            # that arrives through a reconfiguration brings its count with it, a fresh optimizer does not reset it
            l.opt_step += 1
            # a layer sharded over its stage (sharding.py): the update runs on this rank's shard of parameters,
            # reduce-scattered gradient and moments; the planes are split after the next all-gather, not here
            l.prepare_gradient_for_optim()
            L.call("oob_adamw_step", C.c_void_p(l.flat_param.data_ptr()), C.c_void_p(l.flat_grad.data_ptr()),
                   C.c_void_p(l.exp_avg.data_ptr()), C.c_void_p(l.exp_avg_sq.data_ptr()),
                   C.c_void_p(l.optimizer_planes_ptr()), l.plane_stride, l.nplanes, l.flat_param.numel(),
                   float(g["lr"]), g["betas"][0], g["betas"][1], g["eps"], g["weight_decay"], l.opt_step, stream)
            if l.sharded:
                l.refresh_planes()    # marks the gathered copy out of date
            self.state[l.flat_param] = {"step": l.opt_step, "exp_avg": l.exp_avg, "exp_avg_sq": l.exp_avg_sq}

    def zero_grad(self) -> None:
        for l in self.layers:
            l.zero_grad()


class WarmupLR:
    def __init__(self, optimizer, warmup_min_lr: float = 0.0, warmup_max_lr: float = 1e-3,
                 warmup_num_steps: int = 1000, last_batch_iteration: int = -1):
        self.optimizer = optimizer
        self.min_lr = float(warmup_min_lr)
        self.max_lr = float(warmup_max_lr)
        self.delta_lr = self.max_lr - self.min_lr
        self.warmup_num_steps = max(2, warmup_num_steps)
        self.inverse_log_warm_up = 1.0 / math.log(self.warmup_num_steps)
        self.last_batch_iteration = last_batch_iteration
        # deepspeed's constructor publishes the pre-start learning rate to the optimizer
        self._set(self.get_lr())

    def _set(self, lr: float) -> None:
        for group in self.optimizer.param_groups:
            group["lr"] = lr
        self._last_lr = [lr]

    def get_lr(self) -> float:
        if self.last_batch_iteration < 0:
            return 0.0
        if self.last_batch_iteration < self.warmup_num_steps:
            gamma = self.inverse_log_warm_up * math.log(self.last_batch_iteration + 1)
        else:
            gamma = 1.0
        return self.min_lr + self.delta_lr * gamma

    def get_last_lr(self):
        return self._last_lr

    def step(self, last_batch_iteration: int | None = None) -> None:
        if last_batch_iteration is None:
            last_batch_iteration = self.last_batch_iteration + 1
        self.last_batch_iteration = last_batch_iteration
        self._set(self.get_lr())
