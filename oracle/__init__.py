"""
oracle/ -- TEST INFRASTRUCTURE ONLY.  Not part of the product.

A CPU (NumPy/SciPy) restatement of the one Dragonfly hot path this repository accelerates:
  dragonfly/utils/general_utils.py  (dist_squared, stable_cholesky, triangular solves, gaussian draws)
  dragonfly/gp/kernel.py            (SE, Matern, Additive, CoordinateProduct kernels)
  dragonfly/gp/gp_core.py           (GP.build_posterior / eval / hallucinated eval / LML / draw_samples)
  dragonfly/opt/gpb_acquisitions.py (UCB, EI, PI, TTEI, TS, Add-UCB, BOCA fidel_to_opt slice)
  dragonfly/utils/oper_utils.py     (random_sample / random_maximise)
Every function cites the reference file:line it follows (paths relative to the reference source tree).

Who may import this package: ONLY tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
`--impl reference` leg -- and there only as the checker or the CPU baseline, never as the thing
measured or shipped.  dragonfly_b200/ (the product) must never import it; the product fails loudly
when libdfb200.so is missing (dragonfly_b200/_lib.py).

Parity status: PINNED.  oracle/gp_oracle.py is checked (tests/test_oracle_golden.py) against
  (1) the known-answer vectors the reference's own unit tests hold for this path
      (unittest_general_utils.py:26-35, unittest_kernel.py:37-151), restated in tests/golden/, and
  (2) outputs of the UNMODIFIED reference itself, imported from its source tree ($DRAGONFLY_REF) with
      oracle/ref_shim/sitecustomize.py (NumPy-2 aliases only) by tests/golden/make_golden*.py; the resulting
      fixtures are committed under tests/golden/*.npz.  Nothing here reads the reference at run time.
"""
