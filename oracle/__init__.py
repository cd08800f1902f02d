"""CPU oracle for the Oobleck pipeline-execution hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``oobleck_b200/`` may import this
package; only ``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` /
``--impl reference`` legs of ``bench.py`` do, and only as the checker / the
reported CPU baseline -- never as the thing shipped.

What it restates (reference = SymbioticLab/Oobleck @ 3b7a0c2f, never copied):

* ``schedule.py``     -- oobleck/execution/pipeline.py:24-84 (``OobleckPipelineSchedule.steps``)
                         on top of deepspeed ``TrainSchedule`` index math (third party,
                         deepspeed>=0.8.1, not vendored; restated from its published algorithm).
* ``gpt2.py``         -- the HF GPT-2 stage layers produced by oobleck/module/sharding.py:12-18
                         (embedding | one GPT2Block per layer | ln_f + lm_head + shifted CE),
                         plain torch fp32.  Pinned against ``transformers`` 5.5 GPT2LMHeadModel
                         (the third-party module that holds the arithmetic) in
                         tests/test_oracle_gpt2.py.
* ``bookkeeping.py``  -- pipeline_template.h:57-84 (rank grid), pipeline.py:565-623 (wiring),
                         engine.py:363-412 (DP grid), engine.py:91-180,311-360 (reconfiguration
                         policy), dataloader.py:43-100 (sampler), utils.py:4-18 (dtype ids).
* ``optim.py``        -- torch AdamW(fused) arithmetic + deepspeed WarmupLR as the reference
                         constructs them (pipeline.py:117-127).

* ``_ref/``          -- not a restatement: the REFERENCE's own C++ planner module (``pipeline_template``,
                         oobleck/csrc/planning/{pipeline_template.cpp,bind.cpp}) built by ``make -C oracle``
                         from the sources of a reference checkout (OOBLECK_REFERENCE), with single-threaded
                         stand-ins (``shims/``) for cppcoro and oneTBB, which this image lacks.  It pins the
                         product's template search and ``get_rank_grid`` (tests/test_planner_vs_reference.py,
                         golden vectors tests/golden/planner.json).  Git-ignored; built by
                         ``__graft_entry__.build()`` when OOBLECK_REFERENCE is set.

Parity pins: the integer bookkeeping is pinned by golden vectors generated from the
reference's own Python (tests/golden/gen_golden.py imports the reference checkout with the missing
third-party modules stubbed) plus the tables of the reference's tests
(tests/execution/test_reconfiguration.py:151-398, tests/execution/test_engine.py:135-225).
Floating point: pinned against HF transformers (see above); the deepspeed schedule helper
math is "parity unpinned" (deepspeed is not installable here) and says so in DESIGN.md.
"""
