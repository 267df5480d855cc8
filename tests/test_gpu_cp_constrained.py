"""
Constrained Cartesian-product domains on the device (-m gpu): dfb_constraint_status byte for byte against its NumPy
oracle (constraint_ref.py) on 10^6 rows per program, surface, 1-ulp, NaN and Inf rows included; dfb_compact_rows'
order, indices and count; the parity draw against the unmodified reference (golden cp_constrained.npz); device-mode
draws that satisfy the constraints and reproduce from their seed; and the refusals.
"""
import json
from argparse import Namespace

import numpy as np
import pytest

from conftest import load_golden
import constraint_ref as CR
import cp_constrained_ref as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def G():
  import torch
  assert torch.cuda.is_available(), 'these tests need a CUDA device'
  from dragonfly_b200 import gpb_acquisitions, device, _lib, constraints
  return Namespace(acq=gpb_acquisitions, device=device, lib=_lib, cons=constraints, torch=torch,
                   post=device.DevicePosterior(64))


def _rows(G, parts, m, seed):
  np.random.seed(seed)
  _, draws = G.acq.draw_cp_candidates(parts, m)
  X = G.acq._level_rows(draws)
  k = m // 10
  X[:k, 0] = 0.25 - X[:k, 1] * X[:k, 2] + X[:k, 3] / 3                  # on a surface of 'exact'
  X[k:2 * k, 0] = np.nextafter(X[:k, 0], 2.0)
  X[2 * k:3 * k, 2] = 1.5 - np.sqrt(X[2 * k:3 * k, 0] ** 2 + X[2 * k:3 * k, 1] ** 2)     # ... of the fixture's norm
  X[3 * k:4 * k, 2] = np.nextafter(X[2 * k:3 * k, 2], -2.0)
  X[4 * k:4 * k + 50, 0] = np.nan
  X[4 * k + 50:4 * k + 100, 2] = np.inf
  X[4 * k + 100:4 * k + 150, 1] = -np.inf
  X[4 * k + 150:4 * k + 200, 4] = np.nan
  return X


@pytest.mark.parametrize('name', sorted(F.PROGRAMS))
def test_status_kernel_equals_oracle(G, name):
  dom = F.make_domain(F.PROGRAMS[name])
  parts = G.acq._cp_parts(dom, F.make_kernel())
  f = G.cons.compile_filter(dom, parts, levels=True)
  X = _rows(G, parts, 1000000, 21)
  st, counts = G.post.constraint_status(f.desc(), G.torch.from_numpy(X).cuda())
  ref = CR.status(f, X)
  got = st.cpu().numpy()
  assert np.array_equal(got, ref), (name, np.flatnonzero(got != ref)[:10])
  assert counts == [int(np.sum(ref == k)) for k in range(3)]


@pytest.mark.parametrize('m', [0, 1, 1023, 1024, 1025, 5000, 300001, (1 << 21) + 77])
@pytest.mark.parametrize('pattern', ['none', 'all', 'random'])
def test_compaction(G, m, pattern):
  rng = np.random.RandomState(m)
  X = rng.standard_normal((m, 5))
  st = {'none': np.zeros(m), 'all': np.ones(m), 'random': rng.randint(0, 3, m)}[pattern].astype(np.uint8)
  Xd, sd = G.torch.from_numpy(X).cuda(), G.torch.from_numpy(st).cuda()
  rows, idx = G.post.compact_rows(Xd, sd, keep=1, idx_base=7)
  sel = np.flatnonzero(st == 1)
  np.testing.assert_array_equal(idx.cpu().numpy(), sel + 7)
  np.testing.assert_array_equal(rows.cpu().numpy().reshape(-1, 5), X[sel])


@pytest.mark.parametrize('k', range(5))
def test_parity_draw_reproduces_the_reference(G, k):
  g = load_golden('cp_constrained')
  run = json.loads(str(g['runs']))[k]
  if run['kind'] != 'rand':
    pytest.skip('a single sample_from_cp_domain call is checked on the host')
  dom = F.make_domain(F.CONSTRAINTS if run['which'] == 'all' else F.TIGHT)
  parts = G.acq._cp_parts(dom, F.make_kernel())
  np.random.seed(run['seed'])
  source, seed = G.acq._cp_candidate_source(G.post, lambda t: t, parts, run['M'], 'numpy', domain=dom)
  assert seed is None and source.hi == run['count']
  assert [F.jval(source.point(i, None)) for i in range(source.hi)] == run['points']
  F.check_state(g, k)
  assert np.all(np.isfinite(source.fill(0, source.hi, None).cpu().numpy()))


def test_device_mode_keeps_constrained_points_and_reproduces(G):
  dom = F.make_domain(F.CONSTRAINTS)
  parts = G.acq._cp_parts(dom, F.make_kernel())
  np.random.seed(5)
  src, seed = G.acq._cp_candidate_source(G.post, lambda t: t, parts, 3000, 'device', domain=dom)
  assert src.hi == 3000
  pts = [src.point(i, None) for i in range(0, 3000, 37)]
  assert all(dom.constraints_are_satisfied(p) for p in pts)
  np.random.seed(5)
  src2, seed2 = G.acq._cp_candidate_source(G.post, lambda t: t, parts, 3000, 'device', domain=dom)
  assert seed2 == seed
  assert G.torch.equal(src.fill(0, 3000, None), src2.fill(0, 3000, None))
  # the kept set is the oracle's filter of the same device rows, in row order
  kinds, bounds, n_levels, luts = G.acq._cp_device_layout(parts)
  raw = G.post.fill_mixed_candidates(seed, 0, 20000, kinds, bounds, n_levels)
  coded = G.acq._encode_levels(raw.clone(), luts).cpu().numpy()
  f = G.cons.compile_filter(dom, parts)
  st = f.settle(CR.status(f, coded), lambda i: G.acq._cp_point_from_device_row(parts, raw[i].cpu().numpy()))
  keep = np.flatnonzero(st == 1)[:3000]
  assert len(keep) == 3000
  np.testing.assert_array_equal(src.fill(0, 3000, None).cpu().numpy(), coded[keep])


def _acq_anc(g, dom, run, gp, H, **kw):
  Y, Y2 = np.asarray(g['Y']), np.asarray(g['Y2'])
  a = Namespace(domain=dom, max_evals=run['max_evals'], acq_opt_method=run['method'], t=len(gp.X),
                curr_max_val=float(np.max(Y)), handle_parallel='halluc', eval_points_in_progress=H[:run['halluc']],
                is_mf=False, obj_weights=[0.6, 0.4], reference_point=[float(np.min(Y)), float(np.min(Y2))])
  a.__dict__.update(kw)
  return a


@pytest.mark.parametrize('k', range(11))
def test_acquisitions_reproduce_the_reference(G, k):
  from dragonfly_b200 import multiobjective_gpb_acquisitions as moo
  g = load_golden('cp_constrained')
  run = json.loads(str(g['acq_runs']))[k]
  gp, gp2, H = F.golden_gps(g)
  dom = F.make_domain()
  np.random.seed(run['seed'])
  anc = _acq_anc(g, dom, run, gp, H)
  if run['name'] == 'syn_ucb':
    pts = G.acq.syn.ucb(3, gp, anc)
  elif run['name'] in ('lin_ucb', 'tch_ts'):
    pts = [getattr(moo.asy, run['name'])([gp, gp2], anc)]
  else:
    pts = [getattr(G.acq.asy, run['name'])(gp, anc)]
  assert [F.jval(p) for p in pts] == run['points'], run
  F.check_acq_state(g, k)


@pytest.mark.parametrize('name', ['ei', 'ts', 'lin_ucb', 'tch_ts'])
def test_device_mode_acquisitions_return_constrained_points(G, name):
  from dragonfly_b200 import multiobjective_gpb_acquisitions as moo
  g = load_golden('cp_constrained')
  gp, gp2, H = F.golden_gps(g)
  dom = F.make_domain()
  run = dict(max_evals=2000, method='rand', halluc=0)
  picks = []
  for _ in range(2):
    np.random.seed(9)
    anc = _acq_anc(g, dom, run, gp, H, candidate_rng='device')
    pt = getattr(moo.asy, name)([gp, gp2], anc) if name in ('lin_ucb', 'tch_ts') else getattr(G.acq.asy, name)(gp, anc)
    assert dom.constraints_are_satisfied(pt)
    picks.append(F.jval(pt))
  assert picks[0] == picks[1]


def test_refusals(G):
  dom = F.make_domain(F.CONSTRAINTS)
  a = Namespace(domain=dom, max_evals=10, acq_opt_method='ga', t=5, handle_parallel='halluc',
                eval_points_in_progress=[], is_mf=False, candidate_rng='device', curr_max_val=0.0)
  gp, _, _ = F.golden_gps(load_golden('cp_constrained'))
  with pytest.raises(NotImplementedError):                     # the device GA
    G.acq.asy.ei(gp, a)
  import dragonfly_b200.gpb_acquisitions as acq_mod
  orig = acq_mod._shard_info
  acq_mod._shard_info = lambda: (0, 2, None)
  try:
    class _GP(object):
      kernel = F.make_kernel()
    with pytest.raises(NotImplementedError):
      acq_mod._cp_fused_maximise(_GP(), Namespace(domain=dom, max_evals=10), None)
  finally:
    acq_mod._shard_info = orig
