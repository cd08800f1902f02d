"""Template search: this repo's planner (csrc/planning/template_search.cpp behind the C ABI) next to the reference's own
C++ planner (oracle/_ref, built by ``make -C oracle`` from the reference's oobleck/csrc/planning with single-threaded
stand-ins for cppcoro / oneTBB), on the same host core, same random layer profile.

    python tools/planner_timing.py [layers nodes gpus_per_node [reference_budget_s]]

Prints one JSON line per configuration: seconds for both, whether the templates are identical.  The reference run is
bounded (it is a child process that is killed at the budget): its search visits every stage count up to the number of
layers for every node count before it finds most of them infeasible, which this repo's search cuts at the root
(stages > nodes x GPUs per node can never bottom out); the results are the same wherever both finish.
"""
import json
import multiprocessing as mp
import os
import random
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def rows(layers, seed=0):
    rnd = random.Random(seed)
    return [(rnd.uniform(1, 2), rnd.uniform(2, 4)) for _ in range(layers)]


def profile(mod, layers):
    return mod.LayerExecutionResults([
        mod.LayerExecutionResult(i, f, b, {g + 1: 0.05 * (g + 1) for g in range(8)}, {n + 1: 0.1 for n in range(64)},
                                 (1024, 1024)) for i, (f, b) in enumerate(rows(layers))])


def shapes(templates):
    return [(t._num_nodes, [(list(s._layer_indices), s._num_gpus) for s in t.get_stages()]) for t in templates]


def reference_child(layers, nodes, gpn, q):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    import pipeline_template as R
    devnull = os.open(os.devnull, os.O_WRONLY)
    os.dup2(devnull, 1)                      # the module narrates on std::cout
    t0 = time.perf_counter()
    ts = R.PipelineTemplateGenerator().create_pipeline_templates(profile(R, layers), (1, nodes), gpn)
    q.put((time.perf_counter() - t0, shapes(ts)))


def main():
    from oobleck_b200.planning import pipeline_template as P
    args = [int(a) for a in sys.argv[1:4]]
    budget = float(sys.argv[4]) if len(sys.argv) > 4 else 120.0
    configs = [tuple(args)] if len(args) == 3 else [(14, 4, 1), (26, 4, 1), (34, 5, 1), (20, 4, 4), (50, 8, 1)]
    for layers, nodes, gpn in configs:
        t0 = time.perf_counter()
        mine = shapes(P.PipelineTemplateGenerator().create_pipeline_templates(profile(P, layers), (1, nodes), gpn))
        ours = time.perf_counter() - t0
        q = mp.get_context("spawn").Queue()
        p = mp.get_context("spawn").Process(target=reference_child, args=(layers, nodes, gpn, q))
        p.start()
        p.join(budget)
        note = None
        if p.is_alive():
            p.kill()
            p.join()
            ref, same, note = None, None, f"not finished within {budget:.0f} s"
        elif p.exitcode != 0:
            ref, same, note = None, None, f"reference planner died (exit code {p.exitcode})"
        else:
            ref, theirs = q.get(timeout=30)
            same = theirs == mine
        print(json.dumps({"layers": layers, "node_range": [1, nodes], "gpus_per_node": gpn, "this_repo_s": round(ours, 4),
                          "reference_s": None if ref is None else round(ref, 4),
                          "reference_note": note,
                          "identical_templates": same, "host_threads": 1}), flush=True)


if __name__ == "__main__":
    main()
