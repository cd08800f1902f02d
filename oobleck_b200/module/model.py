"""``OobleckModel``: the stage-layer list the planner, profiler and pipeline consume.

Mirrors oobleck/module/model.py:39-91 (same constructor, same public attributes) but does not trace a HF module
with torch.fx: for the GPT family the fx split points (oobleck/module/sharding.py:15-18) always yield
``L + 2`` layers -- embedding | one GPT2Block each | ln_f + lm_head + loss -- so the layer list is written down
directly as light-weight :class:`StageLayerSpec` records.  The arithmetic of each layer kind lives in the CUDA
library (oobleck_b200/csrc/stage.cu); ``oobleck_b200.execution.layer.Layer`` materialises a spec on a GPU.

Only ``gpt2``-type models are in scope (BASELINE.json north_star); other families raise.
"""
from __future__ import annotations

import math
import random
from dataclasses import dataclass
from typing import Any, Optional

import torch

RANDOM_SEED = 42  # model.py:17

lang_models = ["gpt2"]


@dataclass
class GPT2ModelArgs:
    """The subset of HF ``GPT2Config`` the hot path reads (defaults == HF defaults == GPT-2 124M)."""
    model_type: str = "gpt2"
    vocab_size: int = 50257
    n_positions: int = 1024
    n_embd: int = 768
    n_layer: int = 12
    n_head: int = 12
    layer_norm_epsilon: float = 1e-5
    use_cache: bool = False      # model.py:61
    return_dict: bool = False    # model.py:64

    @property
    def num_hidden_layers(self) -> int:
        return self.n_layer

    @classmethod
    def from_args(cls, config_args: dict[str, Any]) -> "GPT2ModelArgs":
        a = dict(config_args)
        if "num_hidden_layers" in a:  # examples/gpt3.yaml:19-22 uses HF's attribute_map alias
            a["n_layer"] = a.pop("num_hidden_layers")
        known = {k: v for k, v in a.items() if k in cls.__dataclass_fields__}
        return cls(**known)


@dataclass(frozen=True)
class StageLayerSpec:
    """One fx shard.  ``kind``: 'embed' (shard 0), 'block' (shards 1..L), 'head' (shard L+1)."""
    index: int
    kind: str
    n_embd: int
    n_head: int
    n_positions: int
    vocab_size: int
    n_layer: int
    layer_norm_epsilon: float

    def param_shapes(self) -> list[tuple[str, tuple[int, ...]]]:
        """Names/shapes in HF ``module.parameters()`` order == FlatParamHandle flatten order (layer.py:96-111)."""
        E, V, P = self.n_embd, self.vocab_size, self.n_positions
        if self.kind == "embed":
            return [("wte", (V, E)), ("wpe", (P, E))]
        if self.kind == "head":
            return [("ln_f_w", (E,)), ("ln_f_b", (E,)), ("lm_head_w", (V, E))]
        return [("ln_1_w", (E,)), ("ln_1_b", (E,)), ("c_attn_w", (E, 3 * E)), ("c_attn_b", (3 * E,)),
                ("c_proj_w", (E, E)), ("c_proj_b", (E,)), ("ln_2_w", (E,)), ("ln_2_b", (E,)),
                ("c_fc_w", (E, 4 * E)), ("c_fc_b", (4 * E,)), ("mlp_proj_w", (4 * E, E)), ("mlp_proj_b", (E,))]

    @property
    def num_params(self) -> int:
        return sum(math.prod(s) for _, s in self.param_shapes())

    def parameters(self):
        """Meta tensors, for callers that only count/inspect parameters (model.py:86-88, profiler.py)."""
        for _, shape in self.param_shapes():
            yield torch.empty(shape, device="meta")

    def init_flat(self, seed: int = RANDOM_SEED) -> torch.Tensor:
        """Deterministic HF-style initial values as one flat fp32 CPU tensor: N(0, 0.02) weights,
        N(0, 0.02/sqrt(2L)) residual projections, LayerNorm (1, 0), zero biases.  (The reference's
        ``init_tensors`` fills everything with ``torch.rand`` -- layer.py:26-37, "TODO: must use checkpointed
        data" -- which is not a trainable initialisation; SURVEY 7 hard part 2.)"""
        g = torch.Generator().manual_seed(seed * 100003 + self.index)
        parts = []
        for name, shape in self.param_shapes():
            if name.startswith("ln_") and name.endswith("_w"):
                parts.append(torch.ones(shape))
            elif name.endswith("_b"):
                parts.append(torch.zeros(shape))
            elif name in ("c_proj_w", "mlp_proj_w"):
                parts.append(torch.randn(shape, generator=g) * (0.02 / math.sqrt(2 * self.n_layer)))
            else:
                parts.append(torch.randn(shape, generator=g) * 0.02)
        return torch.cat([p.reshape(-1) for p in parts])

    # memory model used by the planner's min-node computation (engine.py:492-507)
    def activation_bytes(self, microbatch: int) -> int:
        M, E = microbatch * self.n_positions, self.n_embd
        if self.kind == "block":
            return M * E * (4 * 4 + 2 * 3 * 4) + M * 3 * E * 4 + M * 4 * E * (4 + 6)
        if self.kind == "head":
            vp = (self.vocab_size + 63) // 64 * 64
            return M * vp * (4 + 6) + M * E * 6
        return M * E * 4


class StageLayer:
    """What ``OobleckModel.layers`` holds: one fx shard as the control plane sees it (planning/profiler.py:66-91 and
    :272-274): an object that ``init_tensors(layer, device)`` can materialise, that survives ``copy.deepcopy`` and
    ``.to("cuda")``, whose ``parameters()`` can be counted and which is CALLABLE -- ``layer(*inputs) -> tuple`` with the
    wire tuples of the fx shards (shard 0: ``(input_ids, attention_mask, labels) -> (hidden, labels)``; block:
    ``(hidden, labels) -> (hidden, labels)``; last: ``(hidden, labels) -> (loss, logits)``).

    Everything static is delegated to the :class:`StageLayerSpec`; the compute is an
    ``oobleck_b200.execution.layer.Layer`` (CUDA kernels through the C ABI) built on first use for the micro-batch
    shape of the call.  There is no CPU path: without a GPU / without the extension the call raises."""

    def __init__(self, spec: StageLayerSpec):
        self.spec = spec
        self._impl = None
        self._device = None

    def __getattr__(self, name):            # kind, n_embd, num_params, init_flat(), param_shapes(), ...
        if name in ("spec", "_impl", "_device"):
            raise AttributeError(name)
        return getattr(self.spec, name)

    def __deepcopy__(self, memo):            # profiler.py:66: copy.deepcopy(layer).to("cuda") -- copies share the spec
        return StageLayer(self.spec)

    def __repr__(self):
        return f"StageLayer({self.spec.kind} #{self.spec.index}, {self.spec.num_params} params)"

    def parameters(self):
        return self.spec.parameters()

    def to(self, device):
        self._device = torch.device(device)
        return self

    def materialise(self, microbatch: int, seq_len: int):
        from ..execution.layer import Layer   # needs CUDA + the extension: fails loudly otherwise
        impl = self._impl
        if impl is None or impl.mb != microbatch or impl.T != seq_len:
            dev = self._device if self._device is not None and self._device.type == "cuda" and \
                self._device.index is not None else None
            self._impl = Layer(self.spec.index, self.spec, None, None, None, microbatch_size=microbatch,
                               num_pipe_buffers=1, workspace=None, seq_len=seq_len, device=dev)
        return self._impl

    def __call__(self, *inputs):
        first = inputs[0]
        impl = self.materialise(int(first.shape[0]), int(first.shape[1]))
        if self.spec.kind == "embed":
            ids, mask, labels = inputs
            args = (ids.to(impl.device).contiguous(), mask, labels.to(impl.device).contiguous())
        else:
            hidden, labels = inputs
            args = (hidden.to(impl.device, torch.float32).contiguous(), labels.to(impl.device).contiguous())
        return tuple(impl(args, buffer_id=0))


class OobleckModel:
    """Same constructor and attributes as oobleck/module/model.py:48-91."""

    def __init__(self, model_name: str, sample_inputs: dict[str, Any], training_args: Optional[Any] = None,
                 model_tag: Optional[str] = None, config_args: Optional[dict[str, Any]] = None):
        random.seed(RANDOM_SEED)                          # model.py:56-57
        torch.default_generator.manual_seed(RANDOM_SEED)
        if not any(key in model_name for key in lang_models):
            raise NotImplementedError(
                f"{model_name}: only GPT-2-type models are on the CUDA hot path (north_star); "
                "bert/t5/vit/resnet split points (sharding.py:19-43) are out of scope")
        config_args = dict(config_args or {})
        config_args["use_cache"] = False                 # model.py:61-64
        config_args["return_dict"] = False
        cfg = GPT2ModelArgs.from_args(config_args)
        assert cfg.n_embd % cfg.n_head == 0

        self.sample_inputs = sample_inputs
        self.trace_input_names = list(sample_inputs.keys())
        common = dict(n_embd=cfg.n_embd, n_head=cfg.n_head, n_positions=cfg.n_positions, vocab_size=cfg.vocab_size,
                      n_layer=cfg.n_layer, layer_norm_epsilon=cfg.layer_norm_epsilon)
        kinds = ["embed"] + ["block"] * cfg.n_layer + ["head"]   # sharding.py:15-18 => L + 2 shards
        self.layers = [StageLayer(StageLayerSpec(index=i, kind=k, **common)) for i, k in enumerate(kinds)]
        self.model_name = model_name
        self.model_tag = model_tag
        self.total_num_params = sum(layer.num_params for layer in self.layers)
        self.training_args = training_args
        self.model_args = cfg
