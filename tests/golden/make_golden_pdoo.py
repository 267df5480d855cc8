"""
Generates tests/golden/pdoo.npz by running the UNMODIFIED reference's PDOO maximiser
(dragonfly/utils/oper_utils.py:257-271 -> dragonfly/utils/doo.py) on analytic objectives.  Authoring container:

    PYTHONDONTWRITEBYTECODE=1 PYTHONPATH=oracle/ref_shim:$DRAGONFLY_REF python -W ignore tests/golden/make_golden_pdoo.py

Also records the reference's end-to-end recommendation for asy_ei / asy_ucb with acq_opt_method='pdoo' on the C1 GP
(gpb_acquisitions.py:23-40: the non-vectorised branch of maximise_acquisition).
"""
import os
import sys
from argparse import Namespace

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, '..', '..'))

import dragonfly  # noqa: E402
from dragonfly.utils.oper_utils import pdoo_maximise  # noqa
from dragonfly.utils.doo import DOOFunction, pdoo_wrap  # noqa
from dragonfly.gp.kernel import SEKernel  # noqa
from dragonfly.gp.gp_core import GP  # noqa
from dragonfly.opt import gpb_acquisitions as ref_acq  # noqa
from dragonfly.exd.domains import EuclideanDomain  # noqa
from dragonfly_b200 import synth_data  # noqa

assert dragonfly.__file__.startswith(os.environ['DRAGONFLY_REF'])

OBJECTIVES = {
  'neg_branin': (lambda x: -float(synth_data.branin(np.asarray(x, dtype=np.float64).reshape(1, -1))[0]),
                 [[0, 1], [0, 1]], 300),
  'hartmann6': (lambda x: float(synth_data.hartmann6(np.asarray(x, dtype=np.float64).reshape(1, -1))[0]),
                [[0, 1]] * 6, 400),
  'shifted_1d': (lambda x: float(np.sin(3 * np.asarray(x).ravel()[0]) - 0.1 * np.asarray(x).ravel()[0] ** 2),
                 [[-2, 5]], 120),
  'plateau_3d': (lambda x: float(np.floor(4 * np.asarray(x).ravel()[0]) + np.round(np.asarray(x).ravel()[1], 1)
                             - abs(np.asarray(x).ravel()[2] - 3.0)), [[0, 1], [-1, 1], [2, 4]], 250),
}


def main():
  out = {}
  for name, (f, bounds, evals) in OBJECTIVES.items():
    val, pt, _ = pdoo_maximise(f, bounds, evals)
    _, _, hist = pdoo_wrap(DOOFunction(f, bounds), evals, 1.0, 0.9, 2, 0.8, 1e-3, 0.5, return_history=True)
    out[name + '_val'] = val
    out[name + '_pt'] = pt
    out[name + '_query_pts'] = np.array(hist.query_points)
    out[name + '_query_vals'] = np.array(hist.query_vals)
    print(name, val, pt, len(hist.query_vals))
  # end to end on the C1 GP with the pdoo maximiser
  w = synth_data.make_workload('c1_branin_se_ei', n_cand=10)
  k = w['kernel']
  gp = GP(w['X'], w['Y'], SEKernel(2, k['scale'], k['dim_bandwidths']),
          lambda x: np.array([w['mean_const']] * len(x)), w['noise_var'])
  dom = EuclideanDomain([[0, 1]] * 2)
  for acq in ['ei', 'ucb']:
    anc = Namespace(curr_acq=acq, max_evals=150, t=50, domain=dom, curr_max_val=float(w['Y'].max()),
                    eval_points_in_progress=[], acq_opt_method='pdoo', handle_parallel='halluc', mf_strategy=None,
                    is_mf=False)
    out['e2e_%s_pdoo_point' % acq] = getattr(ref_acq.asy, acq)(gp, anc)
    print(acq, out['e2e_%s_pdoo_point' % acq])
  np.savez_compressed(os.path.join(HERE, 'pdoo.npz'), **out)


if __name__ == '__main__':
  main()
