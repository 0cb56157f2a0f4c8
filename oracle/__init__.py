"""CPU oracle for the EAGLE draft -> verify -> accept hot path.

TEST INFRASTRUCTURE ONLY.  Nothing in ``eagle_b200`` (the product) may import
this package: only ``tests/``, ``__graft_entry__.smoke()`` and the
``cpu_baseline`` / ``--impl reference`` legs of ``bench.py`` use it, and there
only as the checker / CPU baseline, never as the thing shipped.

Parity status: PINNED.  ``oracle/make_golden.py`` imports the unmodified
reference (SafeAILab/EAGLE, a checkout named by EAGLE_REFERENCE), runs its own
``EaModel.eagenerate`` on tiny seeded models and stores every per-phase tensor
under ``tests/golden/``; ``tests/test_oracle_golden.py`` checks this restatement
against those vectors (bit-exact for the integer outputs, bit-exact on the same
host for the floating-point ones).
"""
