"""The engine's dense linear algebra, routine by routine, against a high-precision reference.

`tests/algebra/harness.cu` includes the kernel source and runs one case per warp: the Cholesky factorisations
(`chol_factor`, the register-resident `tn_factor<N>` with its Newton-Hessian assembly), the triangular solves
(`chol_forward`, `chol_back`, `chol_solve_multi`, `tn_forward<N>`, `tn_back<N>`), the products (`symv_row`, `dot_rows`,
`tn_symv_row<N>`, `tn_dot_row<N>`) and `pos_rsqrt`. Every case is staged in the warp's dynamic shared memory, where the
kernels keep their workspace, 16-byte aligned as `build_layout` aligns it.

Two tiers run the same case lists:
  * CPU (`-m "not gpu"`): the harness compiled with g++ -DB200MJ_CPU_EMU, as tests/emu/b200mj_emu.py compiles the engine.
    The emulation has no `rsqrt.approx` seed and no fused multiply-add, so it checks indexing and logic.
  * GPU (`-m gpu`): the harness compiled by nvcc with exactly `__graft_entry__.NVCC_FLAGS`, the arithmetic that ships.

The reference is exact: products and residuals are sums of exact partial products rounded once (`math.fsum` over the
Veltkamp halves of every product, cross-checked against `fractions.Fraction` below; Fractions outright where three
factors meet), solutions and condition numbers come from mpmath at 40 digits. The bounds are backward errors, which
stay sharp whatever the conditioning, and forward errors scaled by the condition number. Every bound is C * n * U with
the one constant C below, whatever the size or the input family.
"""
from __future__ import annotations

import ctypes
import math
import os
import subprocess
import sys
from fractions import Fraction

import mpmath
import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
ALG = os.path.join(HERE, 'algebra')
BUILD = os.path.join(ALG, '_build')
SRC = os.path.join(ALG, 'harness.cu')
DEPS = [SRC, os.path.join(ROOT, 'dm_control_b200', 'csrc', 'b200mj.cu'), os.path.join(HERE, 'emu', 'cuda_emu.h')] + \
       [os.path.join(ROOT, 'include', h) for h in ('b200mj.h', 'b200mj_model_fields.h', 'b200mj_convex.h')]

U = 2.0 ** -53
C = 8                      # every bound below is C * n * U (n: the size, or size + active rows for the Hessian)
MINVAL = 1e-15             # BMJ_MINVAL, include/b200mj_model_fields.h: the pivot clamp
NV_LIST = (6, 9, 12, 18, 22, 27)       # B200MJ_NV_LIST, b200mj.cu
SENT = -7.25e77            # sentinel for workspace the routine must not write

# harness.cu: ops and the parameter row of one case
OP_CHOL, OP_MULTI, OP_TN, OP_PROD, OP_RSQRT = 1, 2, 3, 4, 5
(P_OP, P_N, P_A, P_L, P_DINV, P_B, P_Y, P_FWIN, P_FWOUT, P_BKIN, P_BKOUT, P_K, P_LD, P_XB, P_XX, P_J, P_SD, P_ALIST,
 P_NACT, P_COLBUF, P_NEG, P_V, P_OUT, P_OUT2, P_NROWS) = range(25)
NPAR = 32

mpmath.mp.dps = 40


# ------------------------------------------------------------------------------------------------------------------
# the two builds
# ------------------------------------------------------------------------------------------------------------------
def _stale(target):
  return not os.path.exists(target) or os.path.getmtime(target) < max(os.path.getmtime(d) for d in DEPS)


def _compile(target, cmd):
  if _stale(target):
    os.makedirs(BUILD, exist_ok=True)
    tmp = f'{target}.{os.getpid()}.tmp'
    subprocess.check_call(cmd + ['-o', tmp, SRC])
    os.replace(tmp, target)
  return target


def build_cpu():
  return _compile(os.path.join(BUILD, 'libalgebra_emu.so'),
                  ['g++', '-std=c++20', '-O1', '-fPIC', '-shared', '-pthread', '-x', 'c++', '-DB200MJ_CPU_EMU',
                   '-Wno-unknown-pragmas', '-I' + os.path.join(HERE, 'emu')])


def build_gpu():
  if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
  from __graft_entry__ import NVCC_FLAGS
  return _compile(os.path.join(BUILD, 'libalgebra_sm90a.so'), [os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')] + NVCC_FLAGS)


def _bind(path):
  L = ctypes.CDLL(path)
  vp = ctypes.c_void_p
  L.alg_run.argtypes = [vp, vp, vp, ctypes.c_int, ctypes.c_int, ctypes.c_int]
  assert L.alg_npar() == NPAR
  return L


class CpuTier:
  def __init__(self):
    self.L = _bind(build_cpu())

  def run(self, params, img, warps):
    out = np.empty_like(img)
    rc = self.L.alg_run(params.ctypes.data, img.ctypes.data, out.ctypes.data, img.shape[1], img.shape[0], warps)
    assert rc == 0, rc
    return out


class GpuTier:
  def __init__(self):
    import torch
    if not torch.cuda.is_available():
      pytest.fail('the GPU tier needs a CUDA device')
    self.torch = torch
    self.L = _bind(build_gpu())

  def run(self, params, img, warps):
    t = self.torch
    p = t.as_tensor(params).cuda(); x = t.as_tensor(img).cuda(); y = t.empty_like(x)
    t.cuda.synchronize()
    rc = self.L.alg_run(p.data_ptr(), x.data_ptr(), y.data_ptr(), img.shape[1], img.shape[0], warps)
    assert rc == 0, f'alg_run: CUDA error {rc}'
    return y.cpu().numpy()


_TIERS = {}


@pytest.fixture(scope='module', params=[pytest.param('cpu'), pytest.param('gpu', marks=pytest.mark.gpu)])
def tier(request):
  if request.param not in _TIERS:
    _TIERS[request.param] = CpuTier() if request.param == 'cpu' else GpuTier()
  return _TIERS[request.param]


# ------------------------------------------------------------------------------------------------------------------
# cases: an image of the warp's workspace plus a parameter row
# ------------------------------------------------------------------------------------------------------------------
class Case:
  def __init__(self, op, n, **info):
    self.P = [-1] * NPAR
    self.P[P_OP], self.P[P_N] = op, n
    self.n, self.info, self.parts, self.size = n, info, [], 0

  def put(self, key, data):
    """Append `data` (doubles, or int32 when integer typed) at the next 16-byte boundary; returns its offset."""
    data = np.asarray(data)
    if data.dtype.kind in 'iu':
      words = np.zeros(4 * ((data.size + 3) // 4), np.int32)      # whole 16-byte units
      words[:data.size] = data
      data = words.view(np.float64)
    off = self.size
    self.parts.append((off, np.asarray(data, np.float64).ravel()))
    self.size += 2 * ((data.size + 1) // 2)
    if key is not None:
      self.P[key] = off
    return off

  def alias(self, key, other):
    self.P[key] = self.P[other]


def run_cases(tier, cases, warps=2):
  stride = max(2, max(c.size for c in cases))
  stride += stride % 2
  img = np.full((len(cases), stride), SENT)
  params = np.array([c.P for c in cases], np.int32)
  for i, c in enumerate(cases):
    for off, d in c.parts:
      img[i, off:off + d.size] = d
  out = tier.run(params, img, warps)
  for i, c in enumerate(cases):
    c.out = out[i]
    c.img = img[i]
  return cases


def get(c, key, size):
  return c.out[c.P[key]:c.P[key] + size]


def tri(i):
  return i * (i + 1) // 2


def pack(A):
  return A[np.tril_indices(A.shape[0])]


def unpack(p, n):
  L = np.zeros((n, n))
  L[np.tril_indices(n)] = p
  return L


# ------------------------------------------------------------------------------------------------------------------
# exact reference arithmetic
# ------------------------------------------------------------------------------------------------------------------
def _split(a):
  """Veltkamp: a = hi + lo exactly, each with at most 26 significant bits (so hi*hi, hi*lo, lo*lo are exact)."""
  c = a * 134217729.0
  hi = c - (c - a)
  return hi, a - hi


def exact_dot(a, b, extra=()):
  """sum(a * b) + sum(extra), computed exactly and rounded once."""
  a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
  ah, al = _split(a); bh, bl = _split(b)
  return math.fsum(np.concatenate([ah * bh, ah * bl, al * bh, al * bl, np.asarray(extra, np.float64)]))


def frac_dot(a, b):
  return sum((Fraction(float(x)) * Fraction(float(y)) for x, y in zip(a, b)), Fraction(0))


def llt_residual(L, A):
  """R = L L^T - A (lower triangle, dense), exact and rounded once per entry."""
  n = L.shape[0]
  R = np.zeros((n, n))
  for i in range(n):
    for j in range(i + 1):
      R[i, j] = exact_dot(L[i, :j + 1], L[j, :j + 1], [-A[i, j]])
  return R


def tri_residual(T, x, b):
  """b - T x for a triangular (dense) T, exact; and |T| |x| for the bound."""
  r = np.array([exact_dot(-T[i], x, [b[i]]) for i in range(len(b))])
  return r, np.abs(T) @ np.abs(x)


class MpInverse:
  """A^-1 of a double matrix in mpmath (40 digits), kappa_inf(A), and exact solves A^-1 b rounded to doubles."""

  def __init__(self, A):
    M = A if isinstance(A, mpmath.matrix) else mpmath.matrix(A.tolist())
    n = M.rows
    self.Ai = mpmath.inverse(M)
    norm = lambda X: max(sum(abs(X[i, j]) for j in range(n)) for i in range(n))
    self.kappa = float(norm(self.Ai) * norm(M))

  def solve(self, b):
    return np.array([float(v) for v in self.Ai * mpmath.matrix([float(x) for x in b])])


def assert_componentwise(r, den, bound, what):
  """|r_i| <= bound * den_i for every i (den_i = 0 demands r_i = 0)."""
  bad = np.abs(r) > bound * den
  assert not bad.any(), (what, np.flatnonzero(bad)[:5], float(np.max(np.abs(r) / np.where(den > 0, den, 1) / bound)))


def ulp_distance(a, b):
  ia = np.asarray(a, np.float64).view(np.int64)
  ib = np.asarray(b, np.float64).view(np.int64)
  return np.abs(ia - ib)


# ------------------------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------------------------
def spd(n, cond, rs):
  """Random symmetric positive definite matrix with 2-norm condition number about `cond`."""
  Q = np.linalg.qr(rs.randn(n, n))[0]
  lam = np.logspace(0, -math.log10(cond), n) if n > 1 else np.ones(1)
  A = (Q * lam) @ Q.T
  return (A + A.T) / 2


def scaled(n, rs):
  """D A D with D spanning 1e-6 .. 1e6 in random order: pivots far from 1 (a humanoid's armature next to its masses)."""
  d = np.logspace(-6, 6, n) if n > 1 else np.ones(1)
  d = d[rs.permutation(n)]
  return spd(n, 1e2, rs) * d[:, None] * d[None, :]


FAMILIES = {                 # name -> (matrix generator, condition number) ; 'scaled' is D A D
    'cond1': lambda n, rs: spd(n, 1.0, rs), 'cond1e4': lambda n, rs: spd(n, 1e4, rs),
    'cond1e10': lambda n, rs: spd(n, 1e10, rs), 'scaled': scaled,
}


def chol_case(n, A, rhs, alias, mode, rs):
  """chol_factor (optionally with the ride-along rhs, optionally A aliasing L), then chol_forward and chol_back.
  mode 'out': forward b -> f, back f -> x; 'inplace': forward in place on b, back in place on a second vector b2;
  'chain': forward and back in place on one vector (b -> x, as the engine solves)."""
  c = Case(OP_CHOL, n, A=A, rhs=rhs, alias=alias, mode=mode)
  c.b, c.b2 = rs.randn(n), rs.randn(n)
  c.put(P_A, pack(A))
  if alias:
    c.alias(P_L, P_A)
  else:
    c.put(P_L, np.full(tri(n), SENT))
  c.put(P_DINV, np.full(n, SENT))
  if rhs:
    c.put(P_B, c.b); c.put(P_Y, np.full(n, SENT))
  c.put(P_FWIN, c.b)
  if mode == 'out':
    c.put(P_FWOUT, np.full(n, SENT)); c.alias(P_BKIN, P_FWOUT); c.put(P_BKOUT, np.full(n, SENT))
  elif mode == 'inplace':
    c.alias(P_FWOUT, P_FWIN); c.put(P_BKIN, c.b2); c.alias(P_BKOUT, P_BKIN)
  else:
    c.alias(P_FWOUT, P_FWIN); c.alias(P_BKIN, P_FWIN); c.alias(P_BKOUT, P_FWIN)
  return c


def check_factor(c, A_eff, n_eff, L, dinv):
  """Backward error of L L^T = A_eff, normwise and scaled by the diagonal; dinv[j] L[j][j] = 1."""
  R = llt_residual(L, A_eff)
  nrm = np.linalg.norm(np.tril(R)) / max(np.linalg.norm(np.tril(A_eff)), 1e-300)
  assert nrm <= C * n_eff * U, ('||LL^T - A|| / ||A||', c.info.get('fam'), c.n, nrm / (n_eff * U))
  d = np.sqrt(np.abs(np.diag(A_eff)))
  sc = np.abs(R) / np.outer(d, d)
  assert np.tril(sc).max() <= C * n_eff * U, ('|LL^T - A|_ij / sqrt(A_ii A_jj)', c.info.get('fam'), c.n,
                                                np.tril(sc).max() / (n_eff * U))
  for j in range(len(dinv)):
    e = Fraction(float(dinv[j])) * Fraction(float(L[j, j])) - 1
    assert abs(e) <= 4 * U, ('dinv[j] L[j][j] - 1', c.n, j, float(e) / U)
  return max(nrm, np.tril(sc).max()) / (n_eff * U)


WORST = {}


def note(key, v):
  WORST[key] = max(WORST.get(key, 0.0), float(v))


# ------------------------------------------------------------------------------------------------------------------
# the reference's own exactness
# ------------------------------------------------------------------------------------------------------------------
def test_exact_dot_matches_fraction_sums():
  rs = np.random.RandomState(3)
  for n in (1, 2, 7, 64):
    for scale in (1e-12, 1.0, 1e12):
      a, b, e = rs.randn(n) * scale, rs.randn(n) * np.logspace(-6, 6, n), rs.randn(3)
      ref = frac_dot(a, b) + sum(Fraction(float(x)) for x in e)
      assert exact_dot(a, b, e) == float(ref)


# ------------------------------------------------------------------------------------------------------------------
# chol_factor, chol_forward, chol_back: every n in 1..64
# ------------------------------------------------------------------------------------------------------------------
def _chol_cases(rs):
  cases = []
  for n in range(1, 65):
    for k, fam in enumerate(FAMILIES):
      A = FAMILIES[fam](n, rs)
      # the variants rotate over the families: every n sees both ride-along settings, aliasing and in-place solves
      v = (n + k) % 4
      c = chol_case(n, A, rhs=v in (0, 1), alias=v in (0, 2), mode='inplace' if v in (1, 2) else 'out', rs=rs)
      c.info['fam'] = fam
      cases.append(c)
  return cases


def test_chol_factor_and_substitutions(tier):
  rs = np.random.RandomState(11)
  cases = run_cases(tier, _chol_cases(rs))
  for c in cases:
    n, A = c.n, c.info['A']
    L = unpack(get(c, P_L, tri(n)), n)
    dinv = get(c, P_DINV, n)
    note('chol_factor', check_factor(c, A, n + 1, L, dinv))
    if c.info['rhs']:
      y = get(c, P_Y, n)
      r, den = tri_residual(L, y, c.b)
      assert_componentwise(r, den, C * n * U, ('ride-along y', c.info['fam'], n))
      note('chol_factor ride-along', np.max(np.abs(r) / np.where(den > 0, den, 1)) / (n * U))
    f = get(c, P_FWOUT, n)
    r, den = tri_residual(L, f, c.b)
    assert_componentwise(r, den, C * n * U, ('chol_forward', c.info['fam'], n))
    note('chol_forward', np.max(np.abs(r) / np.where(den > 0, den, 1)) / (n * U))
    x = get(c, P_BKOUT, n)
    r, den = tri_residual(L.T, x, f if c.info['mode'] == 'out' else c.b2)
    assert_componentwise(r, den, C * n * U, ('chol_back', c.info['fam'], n))
    note('chol_back', np.max(np.abs(r) / np.where(den > 0, den, 1)) / (n * U))
    # nothing outside the outputs was written
    used = np.zeros(c.out.size, bool)
    for key, size in ((P_A, tri(n)), (P_L, tri(n)), (P_DINV, n), (P_B, n), (P_Y, n), (P_FWIN, n), (P_FWOUT, n),
                      (P_BKIN, n), (P_BKOUT, n)):
      if c.P[key] >= 0:
        used[c.P[key]:c.P[key] + size] = True
    np.testing.assert_array_equal(c.out[~used], c.img[~used])
    if not c.info['alias']:
      np.testing.assert_array_equal(get(c, P_A, tri(n)), pack(A))


def test_chol_solve_forward_error(tier):
  """factor + forward + back against the exact solve: relative error <= C n U kappa_inf(A), kappa from mpmath."""
  rs = np.random.RandomState(12)
  cases = []
  for n in range(1, 65):
    for fam in ('cond1e4',) if n not in (1, 2, 3, 31, 32, 33, 63, 64) else ('cond1', 'cond1e4', 'cond1e10'):
      c = chol_case(n, FAMILIES[fam](n, rs), rhs=n % 2 == 0, alias=True, mode='chain' if n % 3 else 'out', rs=rs)
      c.info['fam'] = fam
      cases.append(c)
  for c in run_cases(tier, cases):
    ref = MpInverse(c.info['A'])
    xs, x = ref.solve(c.b), get(c, P_BKOUT, c.n)
    err = np.abs(x - xs).max() / np.abs(xs).max()
    assert err <= C * c.n * U * ref.kappa, (c.info['fam'], c.n, err, ref.kappa)
    note('chol solve forward error / kappa', err / (c.n * U * ref.kappa))


def _zero_pivot_case(n, j, diag, rs):
  A = spd(n, 1e3, rs)
  A[j, :] = 0; A[:, j] = 0; A[j, j] = diag
  return A


@pytest.mark.parametrize('diag', [0.0, -1.0, -np.inf])
def test_chol_factor_pivot_clamp(tier, diag):
  """A pivot below BMJ_MINVAL (zero, negative, -inf) is clamped as mju_cholFactor clamps it: with its row and column
  otherwise zero, L[j][j] = sqrt(MINVAL), the column below is zero and the rest is the factor of A with A_jj = MINVAL."""
  rs = np.random.RandomState(13)
  cases = []
  for n in (1, 2, 5, 17, 31, 32, 33, 48, 63, 64):
    for j in sorted({0, n // 2, n - 1}):
      c = chol_case(n, _zero_pivot_case(n, j, diag, rs), rhs=True, alias=n % 2 == 0, mode='chain', rs=rs)
      c.info.update(fam=f'clamp j={j}', j=j)
      cases.append(c)
  for c in run_cases(tier, cases):
    n, j = c.n, c.info['j']
    L = unpack(get(c, P_L, tri(n)), n)
    dinv = get(c, P_DINV, n)
    assert abs(L[j, j] - math.sqrt(MINVAL)) <= 4 * U * math.sqrt(MINVAL), (n, j, L[j, j])
    assert abs(dinv[j] * math.sqrt(MINVAL) - 1) <= 4 * U, (n, j, dinv[j])
    assert not L[j + 1:, j].any() and not L[j, :j].any(), (n, j)
    A_eff = c.info['A'].copy(); A_eff[j, j] = MINVAL
    check_factor(c, A_eff, n + 1, L, dinv)
    x = get(c, P_BKOUT, n)
    assert np.isfinite(x).all() and np.isfinite(get(c, P_Y, n)).all()


NONFINITE = [('nan', 'diag'), ('nan', 'off'), ('inf', 'off'), ('-inf', 'off'), ('inf', 'diag')]


def _poison(A, where, kind, rs):
  n = A.shape[0]
  v = float(kind)
  if where == 'diag':
    j = rs.randint(n); A[j, j] = v
  else:
    i = rs.randint(1, n); j = rs.randint(i); A[i, j] = A[j, i] = v
  return A


@pytest.mark.parametrize('kind,where', NONFINITE)
def test_chol_nonfinite_inputs_stay_visible(tier, kind, where):
  """A NaN anywhere, or an infinity off the diagonal, leaves a non-finite value in the factor and in the solution:
  the pivot clamp must not hide it (the engine's BMJ_WARN_BADQACC looks for it). A +inf pivot leaves a non-finite
  L[j][j]; there 1/L[j][j] is 0 and the solution is finite, as in mju_cholSolve's division by an infinite diagonal."""
  rs = np.random.RandomState(14)
  cases = []
  for n in (1, 2, 4, 9, 31, 32, 33, 64) if where == 'diag' else (2, 4, 9, 31, 32, 33, 64):
    for rhs in (False, True):
      c = chol_case(n, _poison(spd(n, 1e2, rs), where, kind, rs), rhs=rhs, alias=rhs, mode='chain' if rhs else 'out', rs=rs)
      cases.append(c)
  for c in run_cases(tier, cases):
    n = c.n
    assert not np.isfinite(get(c, P_L, tri(n))).all(), (kind, where, n)
    if (kind, where) != ('inf', 'diag'):
      assert not np.isfinite(get(c, P_BKOUT, n)).all(), (kind, where, n)
      if c.info['rhs']:
        assert not np.isfinite(get(c, P_Y, n)).all(), (kind, where, n)


# ------------------------------------------------------------------------------------------------------------------
# chol_solve_multi
# ------------------------------------------------------------------------------------------------------------------
def test_chol_solve_multi(tier):
  """Every column against the exact solve; the padding columns n .. ld-1 of every row are left alone."""
  rs = np.random.RandomState(15)
  ref, cases = {}, []
  for n in (1, 5, 31, 32, 33, 62, 63, 64):
    A = spd(n, 1e4, rs)
    ld = n | 1
    for K in (0, 1, 7, 8, 9, 16, 17):
      for ride in (False, True):
        for alias in (False, True):
          c = Case(OP_MULTI, n, A=A, K=K, ride=ride, alias=alias)
          Bm = np.full((K, ld), SENT)
          Bm[:, :n] = rs.randn(K, n)
          c.B = Bm
          c.xb = rs.randn(n)
          c.put(P_A, pack(A)); c.put(P_L, np.full(tri(n), SENT)); c.put(P_DINV, np.full(n, SENT))
          c.P[P_K], c.P[P_LD] = K, ld
          c.put(P_B, Bm)
          if alias:
            c.alias(P_Y, P_B)
          else:
            c.put(P_Y, np.full(K * ld, SENT))
          if ride:
            c.put(P_XB, c.xb); c.put(P_XX, np.full(n, SENT))
          cases.append(c)
  for c in run_cases(tier, cases):
    n, K, ld = c.n, c.info['K'], c.n | 1
    if id(c.info['A']) not in ref:
      ref[id(c.info['A'])] = MpInverse(c.info['A'])
    inv = ref[id(c.info['A'])]
    X = get(c, P_Y, K * ld).reshape(K, ld)
    sols = list(X[:, :n]) + ([get(c, P_XX, n)] if c.info['ride'] else [])
    rhs = list(c.B[:, :n]) + ([c.xb] if c.info['ride'] else [])
    for k, (x, b) in enumerate(zip(sols, rhs)):
      xs = inv.solve(b)
      err = np.abs(x - xs).max() / np.abs(xs).max()
      assert err <= C * n * U * inv.kappa, (n, K, c.info['ride'], c.info['alias'], k, err / (n * U * inv.kappa))
      note('chol_solve_multi forward error / kappa', err / (n * U * inv.kappa))
    # the padding columns of every row keep the sentinel (B's own when X aliases B); B is read only
    np.testing.assert_array_equal(X[:, n:], SENT)
    if not c.info['alias']:
      np.testing.assert_array_equal(get(c, P_B, K * ld).reshape(K, ld), c.B)
    if K == 0 and not c.info['ride']:      # nothing to solve: nothing is written beyond the factor
      lo = c.P[P_B]
      np.testing.assert_array_equal(c.out[lo:], c.img[lo:])


# ------------------------------------------------------------------------------------------------------------------
# tn_factor<N> (with the Newton-Hessian assembly), tn_back<N>, tn_forward<N>: every N of B200MJ_NV_LIST
# ------------------------------------------------------------------------------------------------------------------
NROWS = 32


def tn_case(N, M, nact, rs, negate=0, alias=False, SD=None):
  LD = N | 1
  c = Case(OP_TN, N, M=M, negate=negate, alias=alias)
  J = np.full((NROWS, LD), SENT)          # the padding column of even N must never be read
  J[:, :N] = rs.randn(NROWS, N)
  SD = rs.uniform(0.01, 100, NROWS) if SD is None else SD
  alist = {0: [], 1: [int(rs.randint(NROWS))], NROWS: list(range(NROWS))}.get(nact)
  if alist is None:                       # a random strictly increasing subset, as the solver builds it
    alist = sorted(rs.choice(NROWS, nact, replace=False).tolist())
  c.J, c.SD, c.alist, c.b, c.b2 = J, SD, alist, rs.randn(N), rs.randn(N)
  c.put(P_A, pack(M)); c.put(P_L, np.full(tri(N), SENT)); c.put(P_DINV, np.full(N, SENT))
  c.put(P_B, c.b); c.put(P_Y, np.full(N, SENT))
  c.put(P_J, J); c.put(P_SD, SD); c.put(P_ALIST, np.array(alist + [-1], np.int32)); c.P[P_NACT] = nact
  c.put(P_COLBUF, np.full(64, SENT))
  c.b3 = rs.randn(N)
  if alias:                               # in place, on a vector of its own: back b3 -> x, forward b2 -> f
    c.put(P_BKIN, c.b3); c.alias(P_BKOUT, P_BKIN)
  else:                                   # back y -> x out of place: x solves the whole system
    c.alias(P_BKIN, P_Y); c.put(P_BKOUT, np.full(N, SENT))
  c.P[P_NEG] = negate
  c.put(P_FWIN, c.b2)
  if alias:
    c.alias(P_FWOUT, P_FWIN)
  else:
    c.put(P_FWOUT, np.full(N, SENT))
  return c


def exact_hessian(c):
  """H = M + sum over active rows of SD_r J_r^T J_r as Fractions."""
  N = c.n
  F = lambda v: Fraction(float(v))
  H = [[F(c.info['M'][i, j]) for j in range(N)] for i in range(N)]
  for r in c.alist:
    Jr = [F(v) for v in c.J[r, :N]]
    s = F(c.SD[r])
    for i in range(N):
      si = s * Jr[i]
      for j in range(i + 1):
        H[i][j] += si * Jr[j]
  for i in range(N):
    for j in range(i):
      H[j][i] = H[i][j]
  return H


@pytest.mark.parametrize('fam', ['cond1e4', 'scaled'])
def test_tn_factor_and_substitutions(tier, fam):
  rs = np.random.RandomState(16)
  cases = []
  for N in NV_LIST:
    for k, nact in enumerate((0, 1, 7, NROWS)):
      cases.append(tn_case(N, FAMILIES[fam](N, rs), nact, rs, negate=k % 2, alias=k in (1, 2)))
  for c in run_cases(tier, cases):
    N, nact = c.n, len(c.alist)
    L = unpack(get(c, P_L, tri(N)), N)
    dinv = get(c, P_DINV, N)
    H = exact_hessian(c)
    # backward error, scaled by the diagonal: |L L^T - H|_ij <= C (N + nact) U sqrt(H_ii H_jj). The assembly rounds
    # each of the nact updates of M, the factorisation adds N, and both are bounded by the diagonal of the exact H.
    worst = 0.0
    for i in range(N):
      for j in range(i + 1):
        r = sum((Fraction(float(L[i, k])) * Fraction(float(L[j, k])) for k in range(j + 1)), Fraction(0)) - H[i][j]
        s = abs(float(r)) / math.sqrt(float(H[i][i]) * float(H[j][j]))
        worst = max(worst, s)
    assert worst <= C * (N + nact) * U, (fam, N, nact, worst / ((N + nact) * U))
    note('tn_factor (Hessian)', worst / ((N + nact) * U))
    for j in range(N):
      assert abs(Fraction(float(dinv[j])) * Fraction(float(L[j, j])) - 1) <= 4 * U, (fam, N, nact, j)
    y = get(c, P_Y, N)
    r, den = tri_residual(L, y, c.b)
    assert_componentwise(r, den, C * N * U, ('tn_factor ride-along y', fam, N, nact))
    x = get(c, P_BKOUT, N) * (-1 if c.info['negate'] else 1)
    yb = c.b3 if c.info['alias'] else y
    r, den = tri_residual(L.T, x, yb)
    assert_componentwise(r, den, C * N * U, ('tn_back', fam, N, nact, c.info['negate']))
    f = get(c, P_FWOUT, N)
    r, den = tri_residual(L, f, c.b2)
    assert_componentwise(r, den, C * N * U, ('tn_forward', fam, N, nact))
    for key, v in (('tn_factor ride-along', tri_residual(L, y, c.b)), ('tn_back', tri_residual(L.T, x, yb)),
                   ('tn_forward', tri_residual(L, f, c.b2))):
      note(key, np.max(np.abs(v[0]) / np.where(v[1] > 0, v[1], 1)) / (N * U))
    if fam == 'cond1e4' and not c.info['alias']:        # the whole solve against the exact Hessian
      Hm = mpmath.matrix(N, N)
      for i in range(N):
        for j in range(N):
          Hm[i, j] = mpmath.mpf(H[i][j].numerator) / H[i][j].denominator
      inv = MpInverse(Hm)
      xs = inv.solve(c.b)
      err = np.abs(x - xs).max() / np.abs(xs).max()
      assert err <= C * (N + nact) * U * inv.kappa, (N, nact, err / ((N + nact) * U * inv.kappa))
      note('tn solve forward error / kappa', err / ((N + nact) * U * inv.kappa))
    np.testing.assert_array_equal(c.J, get(c, P_J, c.J.size).reshape(c.J.shape))      # J is read only


def test_tn_factor_pivot_clamp_and_nonfinite(tier):
  """The register-resident factor clamps and propagates like chol_factor (see the chol_factor tests)."""
  rs = np.random.RandomState(17)
  cases = []
  for N in NV_LIST:
    for diag in (0.0, -1.0, -np.inf):
      j = rs.randint(N)
      c = tn_case(N, _zero_pivot_case(N, j, diag, rs), 0, rs)
      c.info.update(kind='clamp', j=j)
      cases.append(c)
    for kind, where in NONFINITE:
      c = tn_case(N, _poison(spd(N, 1e2, rs), where, kind, rs), 0, rs)
      c.info.update(kind=kind, where=where)
      cases.append(c)
  for c in run_cases(tier, cases):
    N = c.n
    L = unpack(get(c, P_L, tri(N)), N)
    if c.info['kind'] == 'clamp':
      j = c.info['j']
      assert abs(L[j, j] - math.sqrt(MINVAL)) <= 4 * U * math.sqrt(MINVAL), (N, j, L[j, j])
      assert not L[j + 1:, j].any() and not L[j, :j].any(), (N, j)
      assert np.isfinite(get(c, P_Y, N)).all() and np.isfinite(get(c, P_BKOUT, N)).all()
    else:
      assert not np.isfinite(L).all(), (c.info, N)
      if (c.info['kind'], c.info['where']) != ('inf', 'diag'):
        for key in (P_Y, P_BKOUT, P_FWOUT):
          assert not np.isfinite(get(c, key, N)).all(), (c.info, N, key)


# ------------------------------------------------------------------------------------------------------------------
# M v and J v: symv_row / dot_rows (every n in 1..64), tn_symv_row<N> / tn_dot_row<N>
# ------------------------------------------------------------------------------------------------------------------
def _wide(rs, *shape):
  """entries of both signs over twelve decades: the sums cancel"""
  return rs.randn(*shape) * 10.0 ** rs.uniform(-6, 6, shape)


def prod_case(n, rs, tn):
  ld = (n | 1) if tn else n | 1
  c = Case(OP_PROD, n)
  S = _wide(rs, n, n); S = np.tril(S) + np.tril(S, -1).T
  nrows = NROWS if tn else 7
  J = np.full((nrows, ld), SENT)
  J[:, :n] = _wide(rs, nrows, n)
  c.S, c.J, c.v = S, J, _wide(rs, n)
  c.put(P_A, pack(S)); c.put(P_V, c.v); c.put(P_J, J)
  c.put(P_OUT, np.full(n, SENT)); c.put(P_OUT2, np.full(nrows, SENT))
  c.P[P_LD] = 0 if tn else ld
  c.P[P_NROWS] = nrows
  return c


def _check_products(c, what):
  n = c.n
  gamma = n * U / (1 - n * U)
  worst = 0.0
  for vals, rows in ((get(c, P_OUT, n), c.S), (get(c, P_OUT2, c.P[P_NROWS]), c.J[:, :n])):
    for got, row in zip(vals, rows):
      exact = frac_dot(row, c.v)
      absum = float(sum(abs(Fraction(float(a)) * Fraction(float(b))) for a, b in zip(row, c.v)))
      err = abs(Fraction(float(got)) - exact)
      assert err <= Fraction(gamma) * Fraction(absum), (what, n, float(err) / absum / U)
      worst = max(worst, float(err) / absum / (n * U))
  note(what, worst)


def test_symv_row_and_dot_rows(tier):
  rs = np.random.RandomState(18)
  for c in run_cases(tier, [prod_case(n, rs, tn=False) for n in range(1, 65)]):
    _check_products(c, 'symv_row / dot_rows')


def test_tn_symv_row_and_tn_dot_row(tier):
  rs = np.random.RandomState(19)
  for c in run_cases(tier, [prod_case(N, rs, tn=True) for N in NV_LIST for _ in range(3)]):
    _check_products(c, 'tn_symv_row / tn_dot_row')


# ------------------------------------------------------------------------------------------------------------------
# pos_rsqrt
# ------------------------------------------------------------------------------------------------------------------
def rsqrt_inputs():
  xs = [np.logspace(-15, 300, 20000), [MINVAL]]
  p2 = 2.0 ** np.arange(-49, 997)
  xs.append(p2[(p2 >= MINVAL) & (p2 <= 1e300)])
  p4 = 4.0 ** np.arange(-24, 499)
  p4 = p4[(p4 >= MINVAL) & (p4 <= 1e300)]
  xs += [np.nextafter(p4, 0), np.nextafter(p4, np.inf)]
  return np.concatenate([np.asarray(x, np.float64) for x in xs])


def correctly_rounded_rsqrt(x):
  with mpmath.workprec(200):
    return np.array([float(1 / mpmath.sqrt(mpmath.mpf(float(v)))) for v in x])


def test_pos_rsqrt_within_two_ulp(tier):
  """1/sqrt(x) for x in [BMJ_MINVAL, 1e300]: the rsqrt.approx seed plus one cubic step gives full double precision."""
  x = rsqrt_inputs()
  chunk = 2048
  cases = []
  for s in range(0, x.size, chunk):
    part = x[s:s + chunk]
    c = Case(OP_RSQRT, part.size)
    c.put(P_V, part); c.put(P_OUT, np.full(part.size, SENT))
    cases.append(c)
  got = np.concatenate([get(c, P_OUT, c.n) for c in run_cases(tier, cases)])
  d = ulp_distance(got, correctly_rounded_rsqrt(x))
  note('pos_rsqrt (ulp)', d.max())
  assert d.max() <= 2, (x[np.argmax(d)], int(d.max()), int((d > 2).sum()))


def test_report_worst_errors(tier):
  """Runs last in this module: the worst error seen per routine, in units of n U (pos_rsqrt: in ulp)."""
  for k in sorted(WORST):
    print(f'{k:45s} {WORST[k]:8.3f}   (bound {2 if k.startswith("pos_rsqrt") else C})')
