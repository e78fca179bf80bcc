"""oracle/ -- TEST INFRASTRUCTURE ONLY.

CPU restatement of the reference hot path (JonasGeiping/breaching,
``OptimizationBasedAttacker._run_trial`` and what it calls) used to *check* the
sm_90a engine in ``breaching_b200``.  Nothing under ``breaching_b200/`` may
import this package; only ``tests/``, ``__graft_entry__.smoke()`` and the
``cpu_baseline`` / ``--impl reference`` legs of ``bench.py`` do.

Parity pin: ``oracle/restate.py`` is checked against fixtures under
``tests/golden/`` that were produced by running the *unmodified reference*
(imported from /root/reference through ``oracle/refshim.py``) with the script
``tests/golden/make_golden.py`` (committed).  The reference itself ships no tests
or golden vectors for this path (SURVEY.md section 4, section 8c).
"""
