"""TEST INFRASTRUCTURE - not product code.

CPU float64 restatement of the reference learner's V-trace update path
(`learner.py:89-183`, `models.py:12-21,40-49`).  Only `tests/`,
`__graft_entry__.smoke()` and the CPU-baseline / `--impl reference` legs of
`bench.py` may import anything from this package, and only as the checker or the
timed CPU baseline - never on the product path.

Parity pin: the reference ships no tests, golden vectors or known-answer files
(SURVEY.md section 4 / 8c), so the restatement is pinned against outputs of the
reference itself: `oracle/gen_golden.py` imports the unmodified
`learner.py` (with stub `gym` / `pybullet_envs` modules), drives
`Learner._learn()` in-process on seeded batches and writes `tests/golden/*.npz`
(torch version recorded inside); `tests/test_oracle_golden.py` checks both
restatements in this package against those files.
"""
