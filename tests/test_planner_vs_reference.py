"""The planner objects against the reference's OWN C++ planner (oobleck/csrc/planning/pipeline_template.{h,cpp},
execution_result.h, bound by bind.cpp).

* ``tests/golden/planner.json`` was produced by that module itself (tests/golden/gen_planner_golden.py; oracle/Makefile
  builds it from the reference's sources with single-threaded stand-ins for cppcoro / oneTBB): for 17 seeded
  layer profiles -- 1, 2 and 4 GPUs per node, node ranges up to 8, cheap and expensive in-node all-reduce -- the templates
  ``PipelineTemplateGenerator.create_pipeline_templates`` returns and the rank grid of each.  This repo's template search
  (csrc/planning/template_search.cpp behind ``oob_plan_pipeline_templates``) and ``PipelineTemplate.get_rank_grid`` must
  reproduce them: same stage boundaries, same GPUs per stage, iteration time to 1e-12, rank grids equal.
* ``tests/golden/planner_live.json``: that module's answers on further seeded random profiles, hand-built templates and
  stage objects (``python tests/test_planner_vs_reference.py`` regenerates it); the reference's own planner tests
  (tests/planning/test_pipeline_template.py:10-100) run against this package and, when oracle/_ref is built, the module.
"""
import importlib
import json
import os
import random
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from oobleck_b200.planning import pipeline_template as P  # noqa: E402

GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "planner.json")))


def reference_module():
    d = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(d) or not any(f.startswith("pipeline_template") and f.endswith(".so") for f in os.listdir(d)):
        return None
    sys.path.insert(0, d)
    try:
        return importlib.import_module("pipeline_template")
    except ImportError:
        return None
    finally:
        sys.path.remove(d)


def results_from_rows(mod, rows):
    return mod.LayerExecutionResults([
        mod.LayerExecutionResult(i, r["forward"], r["backward"], {int(k): v for k, v in r["allreduce_in_node"].items()},
                                 {int(k): v for k, v in r["allreduce_across_nodes"].items()}, tuple(r["mem_required"]))
        for i, r in enumerate(rows)])


def shape(t):
    return t._num_nodes, [(list(s._layer_indices), s._num_gpus) for s in t.get_stages()]


@pytest.mark.parametrize("case", GOLDEN, ids=[f"seed{c['seed']}-{c['layers']}L-{c['gpus_per_node']}gpn" for c in GOLDEN])
def test_template_search_reproduces_the_reference_planner(case):
    prof = results_from_rows(P, case["profile"])
    mine = P.PipelineTemplateGenerator().create_pipeline_templates(prof, tuple(case["node_range"]), case["gpus_per_node"])
    assert len(mine) == len(case["templates"])
    for got, want in zip(mine, case["templates"]):
        assert got._num_nodes == want["num_nodes"] and got._num_gpus_per_node == want["num_gpus_per_node"]
        assert [(list(s._layer_indices), s._num_gpus) for s in got.get_stages()] == \
               [(s["layer_indices"], s["num_gpus"]) for s in want["stages"]]
        assert got._iteration_time == pytest.approx(want["iteration_time"], rel=1e-12)
        for s, ws in zip(got.get_stages(), want["stages"]):
            assert s._mem_required == ws["mem_required"]          # 6 x parameter bytes + activation bytes per layer
            assert s._forward == pytest.approx(ws["forward"], rel=1e-13)
            assert s._backward == pytest.approx(ws["backward"], rel=1e-13)
        grid = got.get_rank_grid(want["ranks"])
        assert {str(k): v for k, v in grid.items()} == want["rank_grid"]
        assert list(grid) == sorted(grid)                          # std::map order


LIVE = os.path.join(ROOT, "tests", "golden", "planner_live.json")


def rank_grid_cases():
    """60 hand-built templates (seeded): (rows, bounds, gpus, nodes, gpn, ranks) each."""
    rnd = random.Random(5)
    cases = []
    for _ in range(60):
        gpn = rnd.choice([1, 2, 4, 8])
        nodes = rnd.randint(1, 4)
        # stages: every node's GPUs are dealt out in power-of-two pieces
        gpus = []
        for _n in range(nodes):
            left = gpn
            while left:
                g = rnd.choice([x for x in (1, 2, 4, 8) if x <= left])
                gpus.append(g)
                left -= g
        layers = len(gpus) + rnd.randint(0, 6)
        cuts = sorted(rnd.sample(range(1, layers), len(gpus) - 1)) if len(gpus) > 1 else []
        bounds = list(zip([0] + cuts, cuts + [layers]))
        rows = [{"forward": 1.0, "backward": 2.0, "allreduce_in_node": {str(g): 0.1 for g in range(1, 9)},
                 "allreduce_across_nodes": {"1": 0.1}, "mem_required": [8, 8]} for _ in range(layers)]
        ranks = rnd.sample(range(1000), sum(gpus))
        cases.append((rows, bounds, gpus, nodes, gpn, ranks))
    return cases


def live_case(seed):
    """A random profile and node range (seeded): (rows, (lo, hi), gpus per node)."""
    from gen_planner_golden import profile_rows
    rnd = random.Random(seed)
    gpn = rnd.choice([1, 1, 2, 4])
    layers = rnd.randint(3, 11)
    lo = rnd.randint(1, 3)
    hi = rnd.randint(lo, min(layers, lo + 4))
    rows = profile_rows(seed, layers, gpn, rnd.choice([1, 1, 10, 40]))
    return rows, (lo, hi), gpn


STAGE_OBJECT_CASES = [(0, 9, 1), (2, 5, 2), (4, 9, 4), (0, 1, 1)]


def reference_answers(R):
    """What the reference's own planner module computes on the inputs above (stored as tests/golden/planner_live.json
    by ``python tests/test_planner_vs_reference.py`` with oracle/_ref built)."""
    from gen_planner_golden import profile_rows
    out = {"rank_grid": [], "live": {}, "stage_objects": [], "fixture_templates": {}}
    for rows, bounds, gpus, nodes, gpn, ranks in rank_grid_cases():
        rt = R.PipelineTemplate([R.StageExecutionResult(results_from_rows(R, rows), (a, b), g)
                                 for (a, b), g in zip(bounds, gpus)], 1.0, len(rows), nodes, gpn)
        out["rank_grid"].append([[k, v] for k, v in rt.get_rank_grid(ranks).items()])
    for seed in range(100, 124):
        rows, node_range, gpn = live_case(seed)
        theirs = R.PipelineTemplateGenerator().create_pipeline_templates(results_from_rows(R, rows), node_range, gpn)
        out["live"][str(seed)] = {"shapes": [shape(t) for t in theirs],
                                  "iteration_times": [t._iteration_time for t in theirs]}
    profile = fixture_profile(R)
    out["fixture_templates"] = {
        f"{lo},{hi},{gpn}": [template_record(t) for t in
                             R.PipelineTemplateGenerator().create_pipeline_templates(profile, (lo, hi), gpn)]
        for (lo, hi), gpn in FIXTURE_CALLS}
    out["saved_profile"] = saved_profile_files_checked_by(R)
    rows = profile_rows(3, 9, 4)
    for begin, end, gpus in STAGE_OBJECT_CASES:
        b = R.StageExecutionResult(results_from_rows(R, rows), (begin, end), gpus)
        out["stage_objects"].append({"layer_indices": list(b._layer_indices), "num_gpus": b._num_gpus,
                                     "num_layers": b._num_layers, "forward": b._forward, "backward": b._backward,
                                     "mem_required": b._mem_required})
    return out


SAVED_PROFILE_TAG = "saved_profile_test"


def save_test_profile(cache=None):
    """``save_profile_results`` of a 7-layer profile under ``cache`` (default: the reference's location); returns the
    profile, the directory and {file name: text written}."""
    from gen_planner_golden import profile_rows
    from oobleck_b200.planning.profiler import save_profile_results
    mine = results_from_rows(P, profile_rows(21, 7, 4))
    directory = save_profile_results(mine, "gpt2", SAVED_PROFILE_TAG, 3, cache)
    files = {n: (directory / n).read_text() for n in ("mb3.json", "allreduce_in_node.json", "allreduce_across_nodes.json")}
    return mine, directory, files


def saved_profile_files_checked_by(R):
    """The saved profile's files, after the reference's C++ ``get_profile_results`` (it reads
    /tmp/oobleck/profiles/<model>-<tag>/, pipeline_template.cpp:26-79) has read back exactly the profile written."""
    mine, _, files = save_test_profile()
    back = R.get_profile_results("gpt2", SAVED_PROFILE_TAG, 3)
    assert back.size == mine.size == 7
    for a, b in zip(mine.get(), back.get()):
        assert b._index == a._index
        assert b._forward == a._forward and b._backward == a._backward            # JSON round-trips doubles exactly
        assert dict(b._allreduce_in_node) == a._allreduce_in_node
        assert dict(b._allreduce_across_nodes) == a._allreduce_across_nodes
        assert tuple(b._mem_required) == a._mem_required
    return files


def stored_answers():
    with open(LIVE) as f:
        return json.load(f)


def test_rank_grid_of_hand_built_templates_matches_the_reference_module():
    """pipeline_template.h:57-84 directly (before: pinned only through the reference's test tables)."""
    want = stored_answers()["rank_grid"]
    cases = rank_grid_cases()
    assert len(want) == len(cases)
    for (rows, bounds, gpus, nodes, gpn, ranks), w in zip(cases, want):
        mt = P.PipelineTemplate([P.StageExecutionResult(range(a, b), g) for (a, b), g in zip(bounds, gpus)], 1.0,
                                len(rows), nodes, gpn)
        assert [[k, v] for k, v in mt.get_rank_grid(ranks).items()] == w


@pytest.mark.parametrize("seed", range(100, 124))
def test_live_comparison_on_random_profiles(seed):
    """Random profiles through this package's template search against the reference module's answers."""
    want = stored_answers()["live"][str(seed)]
    rows, node_range, gpn = live_case(seed)
    mine = P.PipelineTemplateGenerator().create_pipeline_templates(results_from_rows(P, rows), node_range, gpn)
    assert json.loads(json.dumps([shape(t) for t in mine])) == want["shapes"]
    for a, b in zip(mine, want["iteration_times"]):
        assert a._iteration_time == pytest.approx(b, rel=1e-12)


# ---- the reference's own planner tests (tests/planning/test_pipeline_template.py:10-100), on both modules ---------------
NUM_LAYERS = 10        # the reference's fixture model has 34 stage layers; its own planner needs minutes there on one thread
# (node range, GPUs per node) of every create_pipeline_templates call of the reference's planner tests below
FIXTURE_CALLS = [((1, 1), 1), ((NUM_LAYERS, NUM_LAYERS), 1), ((NUM_LAYERS + 1, NUM_LAYERS + 1), 1), ((2, 8), 1),
                 ((1, 1), 4), ((1, 6), 4)]


def fixture_profile(mod):
    """tests/conftest.py:119-142 get_dummy_profile -- random times, 1 KiB per layer."""
    rnd = random.Random(7)
    return mod.LayerExecutionResults([
        mod.LayerExecutionResult(layer_index=i, forward=rnd.random() + 1e-3, backward=rnd.random() * 3 + 1e-3,
                                 allreduce_in_node={g + 1: rnd.random() for g in range(8)},
                                 allreduce_across_nodes={n + 1: rnd.random() * 4 for n in range(64)},
                                 mem_required=(1024, 1024)) for i in range(NUM_LAYERS)])


def template_record(t):
    return {"num_nodes": t._num_nodes, "num_gpus_per_node": t._num_gpus_per_node, "iteration_time": t._iteration_time,
            "stages": [[list(st._layer_indices), st._num_gpus] for st in t.get_stages()]}


class RecordedReference:
    """The reference planner module's answers to FIXTURE_CALLS on ``fixture_profile``, replayed from
    tests/golden/planner_live.json (``reference_answers`` stores them), for where its compiled module is not built."""

    class LayerExecutionResult:
        def __init__(self, **kwargs):
            self.__dict__.update(kwargs)

    class LayerExecutionResults:
        def __init__(self, results):
            self.size = len(results)

    class PipelineTemplateGenerator:
        def create_pipeline_templates(self, profile, node_range, gpus_per_node):
            import types
            assert profile.size == NUM_LAYERS
            recs = stored_answers()["fixture_templates"][f"{node_range[0]},{node_range[1]},{gpus_per_node}"]
            return [types.SimpleNamespace(
                _num_nodes=r["num_nodes"], _num_gpus_per_node=r["num_gpus_per_node"], _iteration_time=r["iteration_time"],
                get_stages=lambda r=r: [types.SimpleNamespace(_layer_indices=li, _num_gpus=g) for li, g in r["stages"]])
                for r in recs]


def both():
    R = reference_module()
    return [("this repo", P), ("reference", R if R is not None else RecordedReference())]


MODULES = both()


@pytest.fixture(params=MODULES, ids=[w for w, _ in MODULES])
def planner(request):
    """(module, profile): the reference's planner-test fixture profile."""
    mod = request.param[1]
    return mod, fixture_profile(mod)


def test_fixture_templates_match_the_reference():
    """This package's templates for every call of the planner tests below equal the reference module's."""
    want = stored_answers()["fixture_templates"]
    profile = fixture_profile(P)
    for node_range, gpn in FIXTURE_CALLS:
        got = [template_record(t) for t in
               P.PipelineTemplateGenerator().create_pipeline_templates(profile, node_range, gpn)]
        w = want[f"{node_range[0]},{node_range[1]},{gpn}"]
        assert [(g["num_nodes"], g["num_gpus_per_node"], g["stages"]) for g in got] == \
               [(x["num_nodes"], x["num_gpus_per_node"], x["stages"]) for x in w], (node_range, gpn)
        for g, x in zip(got, w):
            assert g["iteration_time"] == pytest.approx(x["iteration_time"], rel=1e-12)


def test_create_pipeline_templates_onegpu(planner):
    mod, profile = planner
    pipeline_templates = mod.PipelineTemplateGenerator().create_pipeline_templates(profile, (1, 1), 1)
    assert len(pipeline_templates) == 1
    assert pipeline_templates[0]._num_nodes == 1
    assert pipeline_templates[0]._num_gpus_per_node == 1
    assert len(pipeline_templates[0].get_stages()) == 1
    assert pipeline_templates[0]._iteration_time > 0


def test_create_pipeline_templates_maxnode(planner):
    mod, profile = planner
    num_nodes = profile.size                     # a property in the binding (bind.cpp:38)
    pipeline_templates = mod.PipelineTemplateGenerator().create_pipeline_templates(profile, (num_nodes, num_nodes), 1)
    assert len(pipeline_templates) == 1
    assert pipeline_templates[0]._num_nodes == num_nodes
    assert pipeline_templates[0]._num_gpus_per_node == 1
    assert len(pipeline_templates[0].get_stages()) == num_nodes
    assert pipeline_templates[0]._iteration_time > 0


def test_create_pipeline_templates_too_many_nodes(planner):
    mod, profile = planner
    num_nodes = profile.size + 1
    assert len(mod.PipelineTemplateGenerator().create_pipeline_templates(profile, (num_nodes, num_nodes), 1)) == 0


def test_create_pipeline_templates_node_range(planner):
    mod, profile = planner
    max_num_nodes = profile.size
    pipeline_templates = mod.PipelineTemplateGenerator().create_pipeline_templates(profile, (2, 8), 1)
    assert 0 < len(pipeline_templates) <= max_num_nodes
    assert 0 < pipeline_templates[0]._num_nodes <= max_num_nodes
    for pipeline_template in pipeline_templates:
        assert pipeline_templates[0]._num_gpus_per_node == 1
        assert 2 <= len(pipeline_template.get_stages()) <= 8
        assert pipeline_template._iteration_time > 0


def test_create_pipeline_templates_multiple_gpus_in_node(planner):
    mod, profile = planner
    pipeline_templates = mod.PipelineTemplateGenerator().create_pipeline_templates(profile, (1, 1), 4)
    assert len(pipeline_templates) >= 1
    assert sum(t._num_gpus_per_node * t._num_nodes for t in pipeline_templates) == 4


def test_create_pipeline_templates_multiple_gpus_in_node_range(planner):
    mod, profile = planner
    pipeline_templates = mod.PipelineTemplateGenerator().create_pipeline_templates(profile, (1, 6), 4)
    assert len(pipeline_templates) >= 1
    for index, template in enumerate(pipeline_templates):
        num_nodes = index + 1
        assert template._num_gpus_per_node == 4
        assert num_nodes == template._num_nodes


def test_stage_objects_built_the_references_way_agree():
    """``StageExecutionResult(layer_results, (begin, end), num_gpus)`` (bind.cpp:40-48): same aggregates as the reference
    module computed."""
    from gen_planner_golden import profile_rows
    rows = profile_rows(3, 9, 4)
    for (begin, end, gpus), b in zip(STAGE_OBJECT_CASES, stored_answers()["stage_objects"]):
        a = P.StageExecutionResult(results_from_rows(P, rows), (begin, end), gpus)
        assert a._layer_indices == b["layer_indices"] and a._num_gpus == b["num_gpus"]
        assert a._num_layers == b["num_layers"] == end - begin
        assert a._forward == pytest.approx(b["forward"], rel=1e-15) and a._backward == pytest.approx(b["backward"], rel=1e-15)
        assert a._mem_required == b["mem_required"]
    assert results_from_rows(P, rows).size == 9
    assert results_from_rows(P, rows).size() == 9          # the stub file's spelling (pipeline_template.pyi:21)



def test_saved_profile_is_what_the_references_get_profile_results_reads(tmp_path):
    """planning/profiler.py::save_profile_results writes, byte for byte, the files the reference's C++
    ``get_profile_results`` was checked to read back as the same profile (``saved_profile_files_checked_by``), by
    default where that reader looks."""
    from oobleck_b200.planning.profiler import get_profile_path
    assert str(get_profile_path("gpt2", SAVED_PROFILE_TAG)) == f"/tmp/oobleck/profiles/gpt2-{SAVED_PROFILE_TAG}"
    _, directory, files = save_test_profile(str(tmp_path))
    assert directory == tmp_path / f"gpt2-{SAVED_PROFILE_TAG}"
    assert files == stored_answers()["saved_profile"]


if __name__ == "__main__":
    R = reference_module()
    assert R is not None, "build oracle/_ref first (make -C oracle REF=<reference checkout>)"
    with open(LIVE, "w") as f:
        json.dump(reference_answers(R), f)
