"""1F1B instruction stream of one pipeline stage.

Same instruction order as ``OobleckPipelineSchedule.steps`` (oobleck/execution/pipeline.py:34-84), which is
deepspeed's ``TrainSchedule`` with the reduce/optimizer instructions stripped.  Instead of a generator walked in
Python every step, the whole per-stage program is computed once at construction into ``self.program`` (a list of
steps, each a list of instruction objects), because the engine replays it every training step.
Pinned bit-exactly against golden vectors from the reference (tests/test_schedule.py).
"""
from __future__ import annotations


class PipeInstruction:
    __slots__ = ("kwargs",)

    def __init__(self, buffer_id: int):
        self.kwargs = {"buffer_id": buffer_id}

    @property
    def buffer_id(self) -> int:
        return self.kwargs["buffer_id"]

    def __repr__(self) -> str:
        return f"{type(self).__name__}(buffer_id={self.buffer_id})"

    def __eq__(self, other) -> bool:
        return type(self) is type(other) and self.kwargs == other.kwargs


class LoadMicroBatch(PipeInstruction): pass      # noqa: E701
class ForwardPass(PipeInstruction): pass         # noqa: E701
class BackwardPass(PipeInstruction): pass        # noqa: E701
class SendActivation(PipeInstruction): pass      # noqa: E701
class RecvActivation(PipeInstruction): pass      # noqa: E701
class SendGrad(PipeInstruction): pass            # noqa: E701
class RecvGrad(PipeInstruction): pass            # noqa: E701


class OobleckPipelineSchedule:
    def __init__(self, micro_batches: int, stages: int, stage_id: int):
        assert 0 <= stage_id < stages and micro_batches >= 1
        self.micro_batches = micro_batches
        self.stages = stages
        self.stage_id = stage_id
        self.prev_stage = stage_id - 1
        self.next_stage = stage_id + 1
        self.program = self._build()

    # deepspeed TrainSchedule.num_pipe_buffers
    def num_pipe_buffers(self) -> int:
        return max(2, min(self.stages - self.stage_id, self.micro_batches))

    def _micro_batch_of(self, step_id: int) -> tuple[int, bool]:
        """(micro-batch id, is_forward) for a schedule step; ids outside [0, M) mean "idle"."""
        half, odd_step = divmod(step_id, 2)
        odd_stage = self.stage_id & 1
        if odd_step == odd_stage:  # even/even or odd/odd: forward slot
            return half - self.stage_id // 2, True
        if odd_stage:              # even step, odd stage: backward slot
            return half - self.stages + (self.stage_id + 1) // 2, False
        return half - self.stages + 1 + self.stage_id // 2, False  # odd step, even stage

    def _build(self) -> list[list[PipeInstruction]]:
        M, nbuf = self.micro_batches, self.num_pipe_buffers()
        has_prev, has_next = self.prev_stage >= 0, self.next_stage < self.stages
        edge_stage = self.stage_id in (0, self.stages - 1)
        program = []
        prev_mb = -1
        for step_id in range(2 * (M + self.stages - 1)):
            mb, fwd = self._micro_batch_of(step_id)
            cur_ok, prev_ok = 0 <= mb < M, 0 <= prev_mb < M
            cmds: list[PipeInstruction] = []
            if fwd:
                if prev_ok and has_prev:
                    cmds.append(SendGrad(prev_mb % nbuf))
                if cur_ok and has_prev:
                    cmds.append(RecvActivation(mb % nbuf))
            else:
                if cur_ok and has_next:
                    cmds.append(RecvGrad(mb % nbuf))
                if prev_ok and has_next:
                    cmds.append(SendActivation(prev_mb % nbuf))
            if edge_stage and fwd and cur_ok:
                cmds.append(LoadMicroBatch(mb % nbuf))
            if cur_ok:
                cmds.append(ForwardPass(mb % nbuf) if fwd else BackwardPass(mb % nbuf))
            program.append(cmds)
            prev_mb = mb
        return program

    def steps(self):
        return iter(self.program)

    def __iter__(self):
        return iter(self.program)


class OobleckEvalSchedule:
    """Forward-only program of one stage (``OobleckPipeline.evaluate``): one step per micro-batch,

        RecvActivation (not on the first stage), LoadMicroBatch (first stage), ForwardPass, SendActivation (not last).

    Every stage receives only from its predecessor and sends only to its successor, in micro-batch order, so the stages
    form a chain that blocking transfers cannot deadlock (tests/test_evaluate_gloo.py simulates it).  Nothing waits for
    a backward, so one pipe buffer suffices: a micro-batch's activations have left the stage before the next arrives."""

    def __init__(self, micro_batches: int, stages: int, stage_id: int):
        assert 0 <= stage_id < stages and micro_batches >= 0
        self.micro_batches = micro_batches
        self.stages = stages
        self.stage_id = stage_id
        first, last = stage_id == 0, stage_id == stages - 1
        self.program = []
        for _ in range(micro_batches):
            cmds: list[PipeInstruction] = []
            if not first:
                cmds.append(RecvActivation(0))
            if first:
                cmds.append(LoadMicroBatch(0))
            cmds.append(ForwardPass(0))
            if not last:
                cmds.append(SendActivation(0))
            self.program.append(cmds)

    def num_pipe_buffers(self) -> int:
        return 1

    def __iter__(self):
        return iter(self.program)
