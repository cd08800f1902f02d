"""Oracle: 1F1B instruction stream.

Restates deepspeed.runtime.pipe.schedule.TrainSchedule helper math (third party, pinned by the
reference at deepspeed>=0.8.1, environment.yml:29; NOT present in the reference checkout -- parity
for the helper math is therefore "unpinned", see oracle/__init__.py) and the reference's own
override ``OobleckPipelineSchedule.steps`` (oobleck/execution/pipeline.py:34-84).

Pure Python, integers only.  Instructions are (name, buffer_id) tuples.
"""
from __future__ import annotations

SEND_GRAD = "SendGrad"
RECV_ACT = "RecvActivation"
RECV_GRAD = "RecvGrad"
SEND_ACT = "SendActivation"
LOAD = "LoadMicroBatch"
FWD = "ForwardPass"
BWD = "BackwardPass"


def num_pipe_buffers(micro_batches: int, stages: int, stage_id: int) -> int:
    # deepspeed TrainSchedule.num_pipe_buffers
    return max(2, min(stages - stage_id, micro_batches))


def step_to_micro_batch(step_id: int, stages: int, stage_id: int) -> tuple[int, bool]:
    # deepspeed TrainSchedule._step_to_micro_batch (+ the four _even/_odd helpers)
    even_step = step_id % 2 == 0
    even_stage = stage_id % 2 == 0
    if even_step and even_stage:
        return step_id // 2 - stage_id // 2, True
    if (not even_step) and (not even_stage):
        return (step_id - 1) // 2 - stage_id // 2, True
    if even_step and (not even_stage):
        return step_id // 2 - stages + (stage_id + 1) // 2, False
    return (step_id - 1) // 2 - stages + 1 + stage_id // 2, False


def steps(micro_batches: int, stages: int, stage_id: int) -> list[list[tuple[str, int]]]:
    """pipeline.py:34-84, statement by statement."""
    nbuf = num_pipe_buffers(micro_batches, stages, stage_id)
    valid_mb = lambda m: 0 <= m < micro_batches
    valid_stage = lambda s: 0 <= s < stages
    prev_stage, next_stage = stage_id - 1, stage_id + 1

    out = []
    prev_mb = -1
    prev_buffer = curr_buffer = None
    for step_id in range(2 * (micro_batches + stages - 1)):
        mb, is_forward = step_to_micro_batch(step_id, stages, stage_id)
        if valid_mb(prev_mb):
            prev_buffer = prev_mb % nbuf
        if valid_mb(mb):
            curr_buffer = mb % nbuf
        cmds = []
        if is_forward:
            if valid_mb(prev_mb) and valid_stage(prev_stage):
                cmds.append((SEND_GRAD, prev_buffer))
            if valid_mb(mb) and valid_stage(prev_stage):
                cmds.append((RECV_ACT, curr_buffer))
        else:
            if valid_mb(mb) and valid_stage(next_stage):
                cmds.append((RECV_GRAD, curr_buffer))
            if valid_mb(prev_mb) and valid_stage(next_stage):
                cmds.append((SEND_ACT, prev_buffer))
        if stage_id == 0 or stage_id == stages - 1:
            if is_forward and valid_mb(mb):
                cmds.append((LOAD, curr_buffer))
        if valid_mb(mb):
            cmds.append((FWD if is_forward else BWD, curr_buffer))
        prev_mb = mb
        out.append(cmds)
    return out
