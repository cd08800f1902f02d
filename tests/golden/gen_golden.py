#!/usr/bin/env python
"""Generate golden vectors for the integer bookkeeping of the hot path FROM THE REFERENCE'S OWN PYTHON.

Run with OOBLECK_REFERENCE naming a checkout of the reference project:

    python tests/golden/gen_golden.py        # rewrites tests/golden/*.json

The reference cannot be imported as is (deepspeed, accelerate, pyomo, simple_parsing, HF-fx ... are not
installed and its C++ planner cannot be built: cppcoro/oneTBB are missing).  This script therefore
installs *inert stubs* for exactly those third-party modules, then imports the reference's
``oobleck.execution.engine`` / ``pipeline`` / ``dataloader`` / ``utils`` modules unmodified from
that checkout and drives the real reference functions:

* ``ReconfigurationEngine.on_reconfigure``      (engine.py:91-180, 311-360)  -> reconfigure.json
* ``DataParallelEngine.__init__`` grouping      (engine.py:363-398)          -> dp_groups.json
* ``OobleckSampler.__iter__``                   (dataloader.py:43-100)       -> sampler.json
* ``OobleckPipelineSchedule.steps``             (pipeline.py:34-84)          -> schedule.json
* ``DTYPE_TO_ID``                               (utils.py:4-18)              -> dtype_ids.json

One stand-in carries logic and is therefore NOT pinned by this script:
  - deepspeed ``TrainSchedule`` helper math (third party)                -> oracle.schedule helpers
The reference's ``steps()`` override itself runs unmodified on top of it.

The C++ planner objects (``PipelineTemplate.get_rank_grid``, pipeline_template.h:57-84) come from the reference's OWN
module when oracle/_ref holds it (``make -C oracle``; the default here) and from the restatement
``oracle.bookkeeping.Template`` otherwise (``--restated-planner`` forces that).  Both produce byte-identical JSON files
(checked by ``--check``, which regenerates into memory with each and compares with what is committed).
"""
from __future__ import annotations

import importlib.abc
import importlib.machinery
import json
import os
import random
import sys
import types
from unittest.mock import MagicMock

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("OOBLECK_REFERENCE", "")
sys.path.insert(0, ROOT)
sys.path.insert(0, REF)

from oracle import bookkeeping as bk  # noqa: E402
from oracle import schedule as osched  # noqa: E402

def real_planner_module():
    """The reference's pybind11 module built by oracle/Makefile, or None."""
    d = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(d):
        return None
    sys.path.insert(0, d)
    try:
        return importlib.import_module("pipeline_template")
    except ImportError:
        return None
    finally:
        sys.path.remove(d)


REAL_PLANNER = None          # set by main()


def make_template(num_layers: int, num_stages: int, num_gpus_per_node: int, num_nodes: int):
    """tests/conftest.py:144-213 (get_dummy_pipeline_template): the same stage / GPU split either as the reference's
    own C++ objects or as the restatement."""
    t = bk.dummy_template(num_layers, num_stages, num_gpus_per_node, num_nodes)
    if REAL_PLANNER is None:
        return t
    R = REAL_PLANNER
    prof = R.LayerExecutionResults([
        R.LayerExecutionResult(i, 0.5, 1.5, {g + 1: 0.1 for g in range(8)}, {n + 1: 0.1 for n in range(64)}, (1024, 1024))
        for i in range(num_layers)])
    stages = [R.StageExecutionResult(prof, (st._layer_indices[0], st._layer_indices[-1] + 1), st._num_gpus)
              for st in t.get_stages()]
    return R.PipelineTemplate(stages, 0.1, num_layers, num_nodes, num_gpus_per_node)


STUB_ROOTS = {"deepspeed", "accelerate", "pyomo", "simple_parsing", "evaluate", "asyncssh", "aiofiles",
              "torchvision", "datasets"}


class _StubLoader(importlib.abc.Loader):
    def create_module(self, spec):
        m = types.ModuleType(spec.name)
        m.__path__ = []  # behave as a package
        m.__getattr__ = lambda name: MagicMock(name=f"{spec.name}.{name}")
        return m

    def exec_module(self, module):
        pass


class _StubFinder(importlib.abc.MetaPathFinder):
    def find_spec(self, fullname, path, target=None):
        if fullname.split(".")[0] in STUB_ROOTS:
            return importlib.machinery.ModuleSpec(fullname, _StubLoader(), is_package=True)
        return None


def install_stubs():
    sys.meta_path.insert(0, _StubFinder())

    # deepspeed.runtime.pipe.schedule: instruction classes + TrainSchedule helper math (stand-in).
    sched = types.ModuleType("deepspeed.runtime.pipe.schedule")

    class PipeInstruction:
        def __init__(self, **kwargs):
            self.name = self.__class__.__name__
            self.kwargs = kwargs

    class BufferOpInstruction(PipeInstruction):
        def __init__(self, buffer_id, **kwargs):
            super().__init__(buffer_id=buffer_id, **kwargs)

    for n in ["OptimizerStep", "ReduceGrads", "ReduceTiedGrads"]:
        setattr(sched, n, type(n, (PipeInstruction,), {}))
    for n in ["LoadMicroBatch", "ForwardPass", "BackwardPass", "SendActivation", "RecvActivation",
              "SendGrad", "RecvGrad"]:
        setattr(sched, n, type(n, (BufferOpInstruction,), {}))

    class TrainSchedule:
        def __init__(self, micro_batches, stages, stage_id):
            self.micro_batches, self.stages, self.stage_id = micro_batches, stages, stage_id
            self.prev_stage, self.next_stage = stage_id - 1, stage_id + 1

        def _valid_micro_batch(self, m):
            return 0 <= m < self.micro_batches

        def _valid_stage(self, s):
            return 0 <= s < self.stages

        def num_pipe_buffers(self):
            return osched.num_pipe_buffers(self.micro_batches, self.stages, self.stage_id)

        def _buffer_idx(self, m):
            return m % self.num_pipe_buffers()

        def _step_to_micro_batch(self, step_id):
            return osched.step_to_micro_batch(step_id, self.stages, self.stage_id)

        def __iter__(self):
            self.it = None
            return self

        def __next__(self):
            if self.it is None:
                self.it = self.steps()
            return next(self.it)

    sched.TrainSchedule = TrainSchedule
    sched.PipeInstruction = PipeInstruction
    sys.modules["deepspeed.runtime.pipe.schedule"] = sched
    import deepspeed.runtime.pipe as _p  # stub package
    _p.schedule = sched

    # C++ planner module stand-in (bookkeeping only)
    if REAL_PLANNER is not None:
        pt = REAL_PLANNER
    else:
        pt = types.ModuleType("oobleck.csrc.planning.pipeline_template")
        pt.PipelineTemplate = bk.Template
        pt.StageExecutionResult = bk.Stage
        for n in ["LayerExecutionResults", "LayerExecutionResult", "PipelineTemplateGenerator", "get_profile_results"]:
            setattr(pt, n, MagicMock(name=n))
    for name in ["oobleck.csrc", "oobleck.csrc.planning"]:
        m = types.ModuleType(name)
        m.__path__ = []
        sys.modules[name] = m
    sys.modules["oobleck.csrc.planning.pipeline_template"] = pt

    # oobleck.execution.dataset pulls in HF datasets + torchvision + network; only its name is needed.
    ds = types.ModuleType("oobleck.execution.dataset")
    ds.OobleckDataset = type("OobleckDataset", (), {})
    sys.modules["oobleck.execution.dataset"] = ds

    # torch 2.0 module paths that moved / HF-fx that was removed: alias or stub (names only).
    import torch.distributed.fsdp._flat_param as _fp
    sys.modules["torch.distributed.fsdp.flat_param"] = _fp
    fx = types.ModuleType("transformers.utils.fx")
    fx.symbolic_trace = MagicMock(name="symbolic_trace")
    sys.modules["transformers.utils.fx"] = fx

    # control-plane dataclasses (simple_parsing based); only the names are needed by engine.py's imports.
    tu = types.ModuleType("oobleck.elastic.training_util")
    tu.OobleckArguments = type("OobleckArguments", (), {})
    sys.modules["oobleck.elastic.training_util"] = tu
    mu = types.ModuleType("oobleck.elastic.message_util")
    mu.DistributionInfo = type("DistributionInfo", (), {})
    sys.modules["oobleck.elastic.message_util"] = mu


def gen_reconfigure(engine_mod, out, seed=1234, per_gpn=40, max_lost=11):
    """Mirror of tests/execution/test_reconfiguration.py's FakeEngine/FakePipeline harness, driven with the
    test's own tables plus random failure sets."""
    NUM_LAYERS = 34  # conftest model: 32 blocks + 2

    class FakePipeline:
        def __init__(self, pid, template, ranks):
            self._pipeline_id, self._template, self._ranks = pid, template, ranks
            self._dataloader = None
            self._global_step = 0
            self.execution = types.SimpleNamespace(_layers=[])
            self.rank_grid = template.get_rank_grid(ranks)

    cases = []
    rng = random.Random(seed)
    for gpn in (1, 2, 4):
        templates = [make_template(NUM_LAYERS, i, gpn, i) for i in range(2, 6)]
        total = sum(i * gpn for i in range(2, 6))
        node_sets = []
        for _ in range(per_gpn):
            k = rng.randint(1, max_lost)
            nodes = sorted(rng.sample(range(14), k))
            node_sets.append(nodes)
        for nodes in node_sets:
            failed = [n * gpn + j for n in nodes for j in range(gpn)]

            eng = types.SimpleNamespace()
            eng._pipeline_templates = templates
            eng._num_gpus_per_node = gpn
            pipelines, used = [], 0
            for pid, t in enumerate(templates):
                n = t._num_nodes * gpn
                pipelines.append(FakePipeline(pid, t, list(range(used, used + n))))
                used += n
            assert used == total
            eng._pipeline = pipelines[0]

            RE = engine_mod.ReconfigurationEngine
            re = RE.__new__(RE)
            re._engine = lambda eng=eng: eng
            re._pipelines = pipelines
            re._min_num_ranks = templates[0]._num_nodes * templates[0]._num_gpus_per_node
            captured = {}

            def fake_reinstantiate(num_instances_set, new_ranks_list, captured=captured):
                captured["ranks"] = [list(r) for r in new_ranks_list]
                captured["templates"] = [(t._num_nodes, n) for t, n in num_instances_set.items()]
                return types.SimpleNamespace()

            re._reinstantiate = fake_reinstantiate
            re._copy_model_states = lambda *a, **k: None
            try:
                re.on_reconfigure(list(failed))
                result = {"ranks": captured["ranks"], "templates": captured["templates"]}
            except RuntimeError as e:
                result = {"error": str(e)}
            except (AttributeError, TypeError) as e:
                # reference dereferences a missing template (None) when a merged list has no matching
                # template size; record as such
                result = {"error": f"{type(e).__name__}"}
            cases.append({"gpus_per_node": gpn, "failed": failed, "result": result})
    out["reconfigure"] = cases


DP_CASES = [(4, [1, 2], [1, 1], [2, 2]), (4, [3], [2], [4]), (4, [3, 5], [2, 1], [4, 5]),
            (1, [4], [2], [4]), (1, [2, 3], [1, 2], [2, 3]), (2, [2, 4], [2, 1], [3, 5])]


def random_dp_cases(seed, count):
    """Heterogeneous pipeline mixes: per template (nodes, stages) with stages a multiple-of-two-friendly GPU split."""
    rng = random.Random(seed)
    cases = []
    while len(cases) < count:
        gpn = rng.choice([1, 2, 4])
        kinds = rng.randint(1, 3)
        nodes = sorted(rng.sample(range(1, 6), kinds))
        nstages, ok = [], True
        for n in nodes:
            total = n * gpn
            choices = [st for st in range(n, min(total, 8) + 1)]
            nstages.append(rng.choice(choices))
        npipes = [rng.randint(1, 3) for _ in nodes]
        try:
            for n, st in zip(nodes, nstages):
                bk.dummy_template(34, st, gpn, n)
        except AssertionError:
            continue
        cases.append((gpn, nodes, npipes, nstages))
    return cases


def gen_dp_groups(engine_mod, out, case_list=None):
    NUM_LAYERS = 34
    import deepspeed.comm as dist
    cases = []
    for gpn, nodes, npipes, nstages in (case_list or DP_CASES):
        templates = [make_template(NUM_LAYERS, s, gpn, n) for n, s in zip(nodes, nstages)]
        pipelines, used = [], 0
        for t, k in zip(templates, npipes):
            for _ in range(k):
                n = t._num_nodes * gpn
                pipelines.append(types.SimpleNamespace(rank_grid=t.get_rank_grid(list(range(used, used + n)))))
                used += n
        groups = []
        dist.new_group = lambda ranks: groups.append(list(ranks)) or len(groups) - 1
        dist.get_rank = lambda *a, **k: 0
        eng = type("Eng", (), {})()
        eng._num_gpus_per_node = gpn
        DPE = engine_mod.DataParallelEngine
        dpe = DPE(eng, pipelines)
        table = {str(l): {str(f): groups[g] for f, g in d.items()} for l, d in dpe._dp_process_groups.items()}
        cases.append({"gpus_per_node": gpn, "nodes": nodes, "num_pipelines": npipes, "stages": nstages,
                      "groups": table, "order": groups})
    out["dp_groups"] = cases


SAMPLER_CASES = [(257, 2, [4], True, 0), (1000, 4, [3, 5], True, 0), (1000, 4, [3, 5], True, 1),
                 (2334, 2, [16, 24, 24], True, 0), (64, 8, [1, 1], False, 0), (100, 3, [2, 1, 4], True, 3)]


def random_sampler_cases(seed, count):
    rng = random.Random(seed)
    return [(rng.randint(1, 700), rng.randint(1, 6), [rng.randint(1, 9) for _ in range(rng.randint(1, 4))],
             rng.random() < 0.7, rng.randint(0, 5)) for _ in range(count)]


def gen_wiring(out, seed, count):
    """The reference's unmodified ``OobleckPipeline.__init__`` / ``initialize_distributed_fsdp`` /
    ``initialize_distributed_pipeline`` (pipeline.py:431-456, 565-617) for every rank of random templates: who is my
    previous / next stage, which per-layer and per-shard-column groups exist (``list(set(ranks))`` order included)."""
    import deepspeed.comm as dist
    from oobleck.execution.pipeline import OobleckPipeline
    rng = random.Random(seed)
    cases = []
    while len(cases) < count:
        gpn = rng.choice([1, 1, 2, 4])
        nodes = rng.randint(1, 5)
        stages = rng.randint(nodes, min(nodes * gpn, 8))
        try:
            bk.dummy_template(34, stages, gpn, nodes)
        except AssertionError:
            continue
        template = make_template(34, stages, gpn, nodes)
        first = rng.randint(0, 40)
        ranks = list(range(first, first + nodes * gpn))
        per_rank = {}
        for me in ranks + [first + nodes * gpn + 3]:                 # every member, and one outsider
            groups = []
            dist.is_initialized = lambda: True
            dist.get_rank = lambda *a, me=me, **k: me
            dist.new_group = lambda r: groups.append(list(r)) or types.SimpleNamespace(ranks=list(r))
            p = OobleckPipeline(0, template, list(ranks), None, 0, None)
            p.initialize_distributed_fsdp()
            layer_groups, groups[:] = [list(g) for g in groups], []
            p.initialize_distributed_pipeline()
            comm = p.communication
            per_rank[str(me)] = {"my_pipeline": p.my_pipeline, "layer_groups": layer_groups,
                                 "shard_groups": [list(g) for g in groups],
                                 "prev": None if comm is None else comm.prev_rank,
                                 "next": None if comm is None else comm.next_rank, "has_comm": comm is not None}
        cases.append({"gpus_per_node": gpn, "nodes": nodes, "stages": stages, "ranks": ranks, "per_rank": per_rank})
    out["wiring"] = cases


def gen_sampler(out, case_list=None):
    from oobleck.execution.dataloader import OobleckSampler
    cases = []
    for n, mbsz, nmb, shuffle, epoch in (case_list or SAMPLER_CASES):
        per = []
        for pi in range(len(nmb)):
            s = OobleckSampler(range(n), mbsz, pi, nmb, 0, epoch, shuffle)
            per.append([list(map(int, b)) for b in s])
        cases.append({"num_samples": n, "microbatch_size": mbsz, "num_microbatches": nmb, "shuffle": shuffle,
                      "epoch": epoch, "batches": per})
    out["sampler"] = cases


def gen_schedule(out):
    from oobleck.execution.pipeline import OobleckPipelineSchedule
    cases = []
    for M, P in [(4, 2), (4, 4), (1, 1), (8, 1), (2, 4), (64, 8), (3, 3), (16, 7), (5, 8)]:
        for s in range(P):
            sch = OobleckPipelineSchedule(micro_batches=M, stages=P, stage_id=s)
            st = [[[type(c).__name__, c.kwargs["buffer_id"]] for c in cmds] for cmds in sch.steps()]
            cases.append({"micro_batches": M, "stages": P, "stage_id": s, "num_pipe_buffers": sch.num_pipe_buffers(),
                          "steps": st})
    out["schedule"] = cases


def generate() -> dict:
    import oobleck.execution.utils as ref_utils
    import oobleck.execution.engine as engine_mod
    out = {}
    gen_reconfigure(engine_mod, out)
    gen_dp_groups(engine_mod, out)
    gen_sampler(out)
    gen_schedule(out)
    out["dtype_ids"] = {str(k).replace("torch.", ""): v for k, v in ref_utils.DTYPE_TO_ID.items()}
    return out


def main():
    global REAL_PLANNER
    check = "--check" in sys.argv
    if "--restated-planner" not in sys.argv:
        REAL_PLANNER = real_planner_module()
    print("planner objects:", "the reference's own module (oracle/_ref)" if REAL_PLANNER is not None
          else "oracle.bookkeeping restatement", file=sys.stderr)
    install_stubs()
    if "--live-reconfigure" in sys.argv:
        # further failure sets through the reference's on_reconfigure, printed instead of stored: SEED COUNT MAX_LOST
        i = sys.argv.index("--live-reconfigure")
        seed, count, max_lost = (int(x) for x in sys.argv[i + 1: i + 4])
        import oobleck.execution.engine as engine_mod
        out = {}
        gen_reconfigure(engine_mod, out, seed, count, max_lost)
        print(json.dumps(out["reconfigure"], separators=(",", ":")))
        return
    if "--live" in sys.argv:
        # random data-parallel layouts and sampler configurations through the reference's own classes: SEED COUNT
        i = sys.argv.index("--live")
        seed, count = int(sys.argv[i + 1]), int(sys.argv[i + 2])
        import oobleck.execution.engine as engine_mod
        out = {}
        gen_dp_groups(engine_mod, out, random_dp_cases(seed, count))
        gen_sampler(out, random_sampler_cases(seed, count))
        gen_wiring(out, seed, count)
        if len(sys.argv) > i + 4:          # ... RECONFIGURE_COUNT MAX_LOST: failure sets through on_reconfigure as well
            gen_reconfigure(engine_mod, out, seed, int(sys.argv[i + 3]), int(sys.argv[i + 4]))
        print(json.dumps(out, separators=(",", ":")))
        return
    out = generate()
    if check:
        bad = []
        for k, v in out.items():
            with open(os.path.join(HERE, f"{k}.json")) as f:
                if f.read() != json.dumps(v, separators=(",", ":")):
                    bad.append(k)
        print("check:", "all golden files reproduced" if not bad else f"DIFFERENT: {bad}", file=sys.stderr)
        sys.exit(1 if bad else 0)
    for k, v in out.items():
        with open(os.path.join(HERE, f"{k}.json"), "w") as f:
            json.dump(v, f, separators=(",", ":"))
        print(k, len(v))


if __name__ == "__main__":
    main()
