"""The oracle stage layer (oracle/layer.py) with the forward-only entry point of ``Layer.evaluate``, so that the
host-side evaluation path (``OobleckEngine.evaluate``: schedule, transfers, result reduction) runs over gloo with the
oracle as stage compute."""
import torch

from oracle.layer import OracleLayer


class OracleEvalWorkspace:
    """What ``evaluate`` needs of an evaluation workspace: the micro-batch shape and the (sum of micro-batch mean
    losses, targets counted) accumulator."""

    def __init__(self, microbatch, seq):
        self.mb, self.T = microbatch, seq
        self.acc = torch.zeros(2, dtype=torch.float64)


class EvalOracleLayer(OracleLayer):
    @classmethod
    def make_eval_workspace(cls, model, microbatch_size, device):
        return OracleEvalWorkspace(microbatch_size, model.layers[0].n_positions)

    def evaluate(self, inputs, eval_ws):
        """Forward only, no autograd record, training state untouched; the head adds into ``eval_ws.acc``."""
        self.unshard_params()
        assert inputs[0].shape[0] == eval_ws.mb
        with torch.no_grad():
            outs = self.module(*inputs)
        if self.spec.kind == "head":
            labels = inputs[1][:, 1:]
            eval_ws.acc[0] += float(outs[0])
            eval_ws.acc[1] += int(((labels >= 0) & (labels < self.spec.vocab_size)).sum())
            return (outs[0],)
        return tuple(o.detach() for o in outs)
