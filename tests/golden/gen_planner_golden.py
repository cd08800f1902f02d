"""Golden vectors for the planner objects from the reference's OWN C++ planner.

    make -C oracle            # builds oracle/_ref/pipeline_template*.so from $OOBLECK_REFERENCE/oobleck/csrc/planning
    python tests/golden/gen_planner_golden.py

Imports the reference's pybind11 module (see oracle/Makefile for how it is built here) and records, for a set of seeded
random layer profiles, what ``PipelineTemplateGenerator.create_pipeline_templates`` returns (stage splits, GPUs per
stage, iteration time) and ``PipelineTemplate.get_rank_grid`` of every template -> tests/golden/planner.json.
The .so needs a checkout of the reference to be built; the JSON does not."""
import io
import json
import os
import random
import sys
from contextlib import redirect_stdout

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))

CASES = [  # (seed, layers, gpus per node, (min nodes, max nodes), scale of the in-node all-reduce times)
    (0, 6, 1, (1, 4), 1), (1, 8, 1, (1, 6), 1), (2, 10, 1, (2, 5), 1), (3, 5, 2, (1, 3), 1), (4, 8, 2, (1, 4), 1),
    (5, 7, 4, (1, 2), 1), (6, 9, 4, (1, 3), 1), (7, 12, 1, (1, 8), 1), (8, 4, 1, (1, 4), 1), (9, 6, 4, (1, 1), 1),
    (10, 9, 2, (2, 4), 1), (11, 14, 1, (3, 7), 1),
    # expensive in-node all-reduce: sharding a stage over a node's GPUs loses against giving the GPUs to more stages
    (12, 6, 2, (1, 2), 40), (13, 8, 4, (1, 2), 40), (14, 7, 4, (1, 1), 15), (15, 9, 2, (1, 3), 25), (16, 10, 4, (2, 2), 8),
]


def profile_rows(seed, layers, gpn, ar_scale=1):
    """Plain-python description of a random profile (also what the product-side test feeds its own classes)."""
    rnd = random.Random(seed)
    rows = []
    for i in range(layers):
        rows.append({"forward": rnd.uniform(0.2, 3.0), "backward": rnd.uniform(0.4, 6.0),
                     "allreduce_in_node": {str(g): ar_scale * rnd.uniform(0.01, 0.3) for g in range(1, gpn + 1)},
                     "allreduce_across_nodes": {str(n + 1): rnd.uniform(0.05, 0.5) for n in range(8)},
                     "mem_required": [rnd.randrange(1, 1 << 20), rnd.randrange(1, 1 << 20)]})
    return rows


def main():
    import pipeline_template as R      # the reference's module
    out = []
    for seed, layers, gpn, node_range, ar_scale in CASES:
        rows = profile_rows(seed, layers, gpn, ar_scale)
        prof = R.LayerExecutionResults([
            R.LayerExecutionResult(i, r["forward"], r["backward"], {int(k): v for k, v in r["allreduce_in_node"].items()},
                                   {int(k): v for k, v in r["allreduce_across_nodes"].items()}, tuple(r["mem_required"]))
            for i, r in enumerate(rows)])
        with redirect_stdout(io.StringIO()):      # python-level prints only; the module's std::cout chatter stays
            templates = R.PipelineTemplateGenerator().create_pipeline_templates(prof, node_range, gpn)
        case = {"seed": seed, "layers": layers, "gpus_per_node": gpn, "node_range": list(node_range), "profile": rows,
                "templates": []}
        for t in templates:
            stages = t.get_stages()
            ranks = list(range(100, 100 + sum(s._num_gpus for s in stages)))
            case["templates"].append({
                "num_nodes": t._num_nodes, "num_gpus_per_node": t._num_gpus_per_node,
                "iteration_time": t._iteration_time,
                "stages": [{"layer_indices": list(s._layer_indices), "num_gpus": s._num_gpus, "forward": s._forward,
                            "backward": s._backward, "mem_required": s._mem_required} for s in stages],
                "ranks": ranks, "rank_grid": {str(k): v for k, v in t.get_rank_grid(ranks).items()}})
        out.append(case)
    path = os.path.join(ROOT, "tests", "golden", "planner.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=0)
    print(f"wrote {path}: {len(out)} cases, {sum(len(c['templates']) for c in out)} templates", file=sys.stderr)


if __name__ == "__main__":
    main()
