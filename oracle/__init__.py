"""TEST INFRASTRUCTURE ONLY -- the parity oracle for the flashy.distrib hot path.

Nothing in ``flashy_b200/`` imports this package.  Only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl reference``
legs may use it, and there only as the checker or the timed CPU baseline.

Two restatements of the reference path live here:

* :mod:`oracle.numeric`  -- single-process arithmetic model (what each collective must
  produce given every rank's inputs).  Used on a 1-GPU box where the W ranks are virtual.
* :mod:`oracle.refdistrib` -- the reference's call sequence over ``torch.distributed``
  (gloo on CPU / NCCL on GPU): one collective per tensor, one divide per tensor, two
  host-synchronising count checks.  Used as the multi-process checker and as the timed
  CPU baseline.

Pinning: both are checked by ``tests/test_oracle.py`` against ``tests/golden/*.npz``,
which were produced by importing the *unmodified* reference ``flashy/distrib.py``
in the build container and running it over gloo with 2, 4 and 8 processes
(``tests/golden/make_golden.py``), and against the known answers of the reference's own
``tests/test_distrib.py`` (mean of 1..8 == 4.5 exactly, broadcast == 1.0 exactly,
count mismatch raises on every rank).
"""
