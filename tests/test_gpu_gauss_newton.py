"""The device Gauss-Newton solve of the Stage-II kernel (``Solver::gauss_newton`` and ``Solver::symv``) against float64, at
the normal equations it was given.

The whole-solve tests see the solve only through converged solutions: rho is computed from the true SSE, so a wrong step
changes the dog-leg's path, not where it ends.  Here one system A dgn = g is solved on its own, in the product's workspace
layout, by the kernel's own device functions: ``tests/tc/gauss_newton_test.cu`` drives them from a test kernel on the GPU
(the pipelined Cholesky with warp 0 on the diagonal blocks and named barrier 1, the right-hand side as row n, the four-warp
backward solve, the three-lanes-per-row ``symv``), and ``mosh2_emu_gauss_newton`` runs the host branch of the same source
(left-looking, one thread) on the same layout.  Before A and g are written, the whole shared memory and global workspace are
filled with NaN bytes, so a read of anything the solve did not write first (identity padding, the kb < 8 masks, the tail of
tmp past npad) shows up as a non-finite result.  The harness kernel is not mosh2_stageii_kernel: it gets its own register
allocation (71-134 registers against the product's 168 / 255), so it pins the GPU branch's algorithm, masks and
synchronisation, not the product binary; the product's own solve runs in the whole-solve tests and in the fallback test
at the end of this file.

Reference (float64 from the A and g the solve was given; float32: the rounded values, exact in float64), D = diag(A_ii)^-1/2:
  eta   = |D (g - A dgn)| / (|DAD| |D^-1 dgn| + |D g|)        (2-norms; residual in extended precision)   <= 8 n u
  fwd   = |D^-1 dgn - x| / |x|, x = (DAD)^-1 D g               (float64 solve + one refinement step)      <= kappa_2(DAD) 8 n u
  symv  |Ag - A g| <= 2 n u |A| |g| entrywise
with u = 2^-24 / 2^-53.  Cholesky is backward stable, so the eta bound holds whatever the conditioning; a dropped update term,
a wrong mask or a wrong block inverse is an O(1) error.  Everything must be finite.

Not positive definite: the kernel gives up on a scaled pivot not above pivot_eps (1e-6 / 1e-13).  A case whose smallest
pivot of the float64 LDL^T of DAD is above 100 pivot_eps must return ok = 1, one below pivot_eps / 100 must return ok = 0;
nothing in between is tested.

Measured maxima as fractions of their bounds (eta, fwd, symv), over every layout and thread count; H100 80GB HBM3 at a
700 W power limit:
                        host twin f32        host twin f64        H100 f32             H100 f64
  every block shape     0.11  0.22  0.22     0.049 0.22  0.29     0.11  0.22  0.22     0.057 0.22  0.29
  larger layouts        0.012 0.023 0.11     0.011 0.029 0.18     0.011 0.012 0.11     0.023 0.029 0.13
  real systems          0.026 0.010 0.13     0.039 0.033 0.17     0.017 0.014 0.17     0.026 0.033 0.18
No bound was widened.
"""
import ctypes as C

import numpy as np
import pytest

from conftest import gpu_solve
from moshpp_b200 import lib
from test_gpu_normal_equations import FAMILIES, PREC, _prepare, emu_lin, gpu_linearize, lin_inputs  # noqa: F401 (emu_lin: a fixture)

U = {'f32': 2.0 ** -24, 'f64': 2.0 ** -53}
PIVOT_EPS = {'f32': 1e-6, 'f64': 1e-13}
KAPPA = {'f32': 1e3, 'f64': 1e8}             # largest kappa_2(DAD) of the synthetic systems
THREADS = {'f32': 384, 'f64': 256}           # the launch bound of mosh2_stageii_kernel
NMAX = 136
# the launcher's range: MOSH2_DEV_BIG (global workspace) and MOSH2_DEV_THREADS
LAYOUTS = [(p, big, t) for p in ('f32', 'f64') for big in (0, 1) for t in ((128, 256, 384) if p == 'f32' else (128, 256))]
STEP1_IN_STEP2 = [6, 8, 9, 63, 64] + list(range(104, 112))


def _bind(fn):
    fn.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.POINTER(lib.ModelDesc), C.c_int32, lib._f64p, lib._f64p, lib._f64p,
                   lib._f64p, C.POINTER(C.c_int32)]
    fn.restype = C.c_int32

    def run(precision, big, threads, desc, A, g):
        """(rc, dgn, Ag, ok); rc = -1: a layout the library would not launch."""
        n = len(g)
        A, g = np.ascontiguousarray(A, dtype=np.float64), np.ascontiguousarray(g, dtype=np.float64)
        dgn, Ag, ok = np.zeros(n), np.zeros(n), C.c_int32(-1)
        rc = fn(PREC[precision], big, threads, C.byref(desc), n, lib._ptr(A, lib._f64p), lib._ptr(g, lib._f64p),
                lib._ptr(dgn, lib._f64p), lib._ptr(Ag, lib._f64p), C.byref(ok))
        assert rc in (0, -1), rc
        return rc, dgn, Ag, ok.value
    return run


@pytest.fixture(scope='module')
def emu_gn():
    from moshpp_b200 import build
    return _bind(C.CDLL(build.build_emu()).mosh2_emu_gauss_newton)


@pytest.fixture(scope='module')
def gpu_gn():
    from moshpp_b200 import build
    return _bind(C.CDLL(build.build_gn_test()).gn_run)


def layout_desc(n2, n1=None):
    """A model that carries only the dimensions that size the solve's workspace: n1 / n2 free variables."""
    d = lib.ModelDesc()
    d.n_joints = d.n_markers = d.kw = 1
    d.n_free1, d.n_free2 = n1 or n2, n2
    return d


# ---- systems ---------------------------------------------------------------------------------------------------------

def rounded(a, precision):
    return a.astype(np.float32).astype(np.float64) if precision == 'f32' else a


def scaled(A):
    """D A D with the kernel's Jacobi scaling (ds = 0 where A_ii <= 0), and D."""
    dg = np.diag(A)
    d = np.where(dg > 0, 1.0 / np.sqrt(np.where(dg > 0, dg, 1.0)), 0.0)
    return A * np.outer(d, d), d


def min_pivot(B):
    """Smallest pivot of the unpivoted float64 LDL^T of B, up to the first one that is not positive."""
    B = B.copy()
    p_min = np.inf
    for k in range(len(B)):
        p = B[k, k]
        p_min = min(p_min, p)
        if p <= 0:
            break
        B[k + 1:, k + 1:] -= np.outer(B[k + 1:, k], B[k + 1:, k]) / p
    return p_min


def spd_system(n, precision, seed, kappa):
    """A = J^T J + a small ridge: J has m = 3M >= n rows, singular values log-spaced down to kappa^-1/2, and columns scaled
    by 10^U(-3, 3), so that the Jacobi scaling matters."""
    rng = np.random.default_rng(seed)
    m = 3 * (n // 3 + 2)
    q1 = np.linalg.qr(rng.normal(size=(m, n)))[0]
    q2 = np.linalg.qr(rng.normal(size=(n, n)))[0]
    s = 10.0 ** rng.uniform(-3, 3, n)
    J = (q1 * np.logspace(0, -0.5 * np.log10(kappa), n)) @ q2.T * s
    A = J.T @ J + 1e-3 / kappa * np.diag(s ** 2)
    A = 0.5 * (A + A.T)
    g = J.T @ rng.normal(size=m)
    return rounded(A, precision), rounded(g, precision)


def diagonal_system(n, precision, seed):
    rng = np.random.default_rng(seed)
    return rounded(np.diag(10.0 ** rng.uniform(-6, 6, n)), precision), rounded(rng.normal(size=n), precision)


def block_shape_systems(precision):
    """Every n from 1 to NMAX (every residue mod 8; the right-hand-side row in warp 0's rows and in the trailing tiles), kappa
    cycling through 1 .. KAPPA, and one diagonal-only A."""
    for n in range(1, NMAX + 1):
        yield n, spd_system(n, precision, n, KAPPA[precision] ** ((n % 4) / 3))
    yield 77, diagonal_system(77, precision, 0)


def not_positive_definite_systems(n, precision, seed):
    """(label, A, g): a zero row and column (ds = 0), rank-deficient J^T J (column c a copy of an earlier column a, so the
    null direction first appears at c) in the first, a middle and the last (short) block, and an indefinite A.  The
    J^T J part is close to the identity after scaling: a pivot that is zero in exact arithmetic stays within a few u of
    zero in float32 too.  Scales are powers of two, so the copies stay exact after rounding."""
    rng = np.random.default_rng(seed)
    m = n + 6
    s = 2.0 ** rng.integers(-10, 11, n)

    def near_identity():
        return np.eye(m, n) + rng.normal(0, 0.3 / np.sqrt(n), (m, n))

    mid = n // 2
    for at in (0, mid, n - 1):
        J = near_identity() * s
        A = J.T @ J
        A[at, :] = 0
        A[:, at] = 0
        yield f'zero row {at}', A, J.T @ rng.normal(size=m)
    for a, c in ((1, 5), (3, mid), (mid, n - 2)):
        J = near_identity()
        J[:, c] = J[:, a]
        sc = s.copy()
        sc[c] = sc[a]
        J = J * sc
        yield f'copy of column {a} at {c}', J.T @ J, J.T @ rng.normal(size=m)
    q = np.linalg.qr(rng.normal(size=(n, n)))[0]
    B = (q * np.r_[-0.5, np.ones(n - 1)]) @ q.T
    B = 0.5 * (B + B.T)
    assert np.diag(B).min() > 0.5
    yield 'indefinite', B * np.outer(s, s), s * rng.normal(size=n)


# ---- measures --------------------------------------------------------------------------------------------------------

def solve_errors(A, g, dgn, Ag, precision):
    """eta / 8nu, fwd / (kappa 8nu), symv / 2nu for one solved system (A, g as the solve was given them)."""
    n, u = len(g), U[precision]
    assert np.isfinite(dgn).all() and np.isfinite(Ag).all()
    B, d = scaled(A)
    Al, gl, xl = A.astype(np.longdouble), g.astype(np.longdouble), dgn.astype(np.longdouble)
    res = (d * (gl - Al @ xl)).astype(np.float64)
    y = dgn / d
    eta = np.linalg.norm(res) / (np.linalg.norm(B, 2) * np.linalg.norm(y) + np.linalg.norm(d * g))
    x = np.linalg.solve(B, d * g)
    x = x + np.linalg.solve(B, (d * gl - B.astype(np.longdouble) @ x.astype(np.longdouble)).astype(np.float64))
    ev = np.linalg.eigvalsh(B)
    kappa = ev[-1] / ev[0]
    fwd = np.linalg.norm(y - x) / np.linalg.norm(x)
    e = dict(eta=eta / (8 * n * u), fwd=fwd / (kappa * 8 * n * u), symv=symv_error(A, g, Ag, precision))
    for k, v in e.items():
        assert v <= 1.0, (n, k, v)
    return e


def symv_error(A, g, Ag, precision):
    n = len(g)
    err = np.abs(Ag.astype(np.longdouble) - A.astype(np.longdouble) @ g.astype(np.longdouble)).astype(np.float64)
    bound = 2 * n * U[precision] * (np.abs(A) @ np.abs(g))
    assert np.isfinite(Ag).all() and (err <= bound).all(), (n, (err - bound).max())
    return float((err / np.maximum(bound, 1e-300)).max())


def expected_ok(A, precision):
    """1 / 0 where the float64 LDL^T of DAD keeps a clear margin to pivot_eps, else None."""
    p = min_pivot(scaled(A)[0])
    return 1 if p > 100 * PIVOT_EPS[precision] else 0 if p < PIVOT_EPS[precision] / 100 else None


def solve_and_check(run, precision, big, threads, desc, A, g, st):
    """Solves one SPD system, checks it and folds its measures into ``st``; False if the layout was refused."""
    assert expected_ok(A, precision) == 1
    rc, dgn, Ag, ok = run(precision, big, threads, desc, A, g)
    if rc == -1:
        return False
    assert ok == 1, len(g)
    for k, v in solve_errors(A, g, dgn, Ag, precision).items():
        st[k] = max(st.get(k, 0.0), v)
    return True


def allow_refusal(precision, big, refused, n_fit_min):
    """Only the float64 shared-memory layout may be refused, and only above a size."""
    if refused:
        assert precision == 'f64' and not big, refused
        assert min(refused) > n_fit_min, refused


def _maxima(st):
    return {k: float('%.2g' % v) for k, v in st.items()}


# ---- the checks, for either back end -----------------------------------------------------------------------------------

def check_block_shapes(run, precision, big, threads):
    st, refused = {}, []
    for n, (A, g) in block_shape_systems(precision):
        if not solve_and_check(run, precision, big, threads, layout_desc(n), A, g, st):
            refused.append(n)
    if refused:        # the layout grows with n: what is refused is a tail
        assert refused == list(range(refused[0], NMAX + 1)), refused
    allow_refusal(precision, big, refused, 64)
    return st


def check_larger_layouts(run, cases, precision, big, threads):
    """A Step-1-sized system in a Step-2-sized layout (n2 = 111), and every family's own (n1, n2) with synthetic systems."""
    st, refused = {}, []
    for n in STEP1_IN_STEP2:
        A, g = spd_system(n, precision, 1000 + n, KAPPA[precision] ** ((n % 4) / 3))
        assert solve_and_check(run, precision, big, threads, layout_desc(111, n), A, g, st) or (precision, big) == ('f64', 0)
    for name in FAMILIES:
        holder = lib.DescHolder(cases(name)['pack'])
        d = holder.desc
        for n in (d.n_free1, d.n_free2):
            A, g = spd_system(n, precision, 2000 + n, KAPPA[precision])
            if not solve_and_check(run, precision, big, threads, d, A, g, st):
                refused.append(n)
    allow_refusal(precision, big, refused, 0)
    return st


def check_not_positive_definite(run, precision, big, threads):
    seen = 0
    for n in (43, 111):
        for label, A, g in not_positive_definite_systems(n, precision, n):
            A, g = rounded(A, precision), rounded(g, precision)
            assert expected_ok(A, precision) == 0, label
            rc, dgn, Ag, ok = run(precision, big, threads, layout_desc(n), A, g)
            if rc == -1:
                allow_refusal(precision, big, [n], 64)
                continue
            assert ok == 0, (n, label)
            symv_error(A, g, Ag, precision)
            seen += 1
    assert seen >= 7


def check_real_systems(run, lins, desc, precision):
    """The normal equations of every linearised frame, solved in the precision they were built in."""
    st = {}
    for A, g in lins:
        exp = expected_ok(A, precision)
        assert exp is not None
        for big in (0, 1):
            rc, dgn, Ag, ok = run(precision, big, THREADS[precision], desc, A, g)
            if rc == -1:
                allow_refusal(precision, big, [len(g)], 0)
                continue
            assert ok == exp
            if ok:
                for k, v in solve_errors(A, g, dgn, Ag, precision).items():
                    st[k] = max(st.get(k, 0.0), v)
    return st


# ---- CPU twin: the host branch of the same source -------------------------------------------------------------------------

@pytest.mark.parametrize('big', [0, 1])
@pytest.mark.parametrize('precision', ['f32', 'f64'])
def test_device_source_solves_every_block_shape(emu_gn, precision, big):
    print(precision, big, _maxima(check_block_shapes(emu_gn, precision, big, THREADS[precision])))


@pytest.mark.parametrize('big', [0, 1])
@pytest.mark.parametrize('precision', ['f32', 'f64'])
def test_device_source_solves_in_larger_layouts(cases, emu_gn, precision, big):
    print(precision, big, _maxima(check_larger_layouts(emu_gn, cases, precision, big, THREADS[precision])))


@pytest.mark.parametrize('big', [0, 1])
@pytest.mark.parametrize('precision', ['f32', 'f64'])
def test_device_source_rejects_systems_that_are_not_positive_definite(emu_gn, precision, big):
    check_not_positive_definite(emu_gn, precision, big, THREADS[precision])


@pytest.mark.parametrize('precision', ['f32', 'f64'])
@pytest.mark.parametrize('step', [1, 2])
@pytest.mark.parametrize('name', FAMILIES)
def test_device_source_solves_the_real_normal_equations(cases, emu, emu_lin, emu_gn, name, step, precision):
    case = cases(name)
    pk, opts = _prepare(case)
    obs, vis, x = lin_inputs(case, emu(case))
    out = emu_lin(pk, opts, obs, vis, x, step, precision)
    holder = lib.DescHolder(pk)
    st = check_real_systems(emu_gn, zip(out['A'], out['g']), holder.desc, precision)
    print(name, step, precision, _maxima(st))


# ---- the CUDA harness and the product kernel ---------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize('precision,big,threads', LAYOUTS)
def test_kernel_solves_every_block_shape(gpu_gn, precision, big, threads):
    print(precision, big, threads, _maxima(check_block_shapes(gpu_gn, precision, big, threads)))


@pytest.mark.gpu
@pytest.mark.parametrize('precision,big,threads', LAYOUTS)
def test_kernel_solves_in_larger_layouts(cases, gpu_gn, precision, big, threads):
    print(precision, big, threads, _maxima(check_larger_layouts(gpu_gn, cases, precision, big, threads)))


@pytest.mark.gpu
@pytest.mark.parametrize('precision,big,threads', LAYOUTS)
def test_kernel_rejects_systems_that_are_not_positive_definite(gpu_gn, precision, big, threads):
    check_not_positive_definite(gpu_gn, precision, big, threads)


@pytest.fixture(scope='module')
def gpu_states():
    cache = {}

    def get(case, name):
        if name not in cache:
            cache[name] = lin_inputs(case, gpu_solve(case, precision='f64'))
        return cache[name]
    return get


@pytest.mark.gpu
@pytest.mark.parametrize('precision', ['f32', 'f64'])
@pytest.mark.parametrize('step', [1, 2])
@pytest.mark.parametrize('name', FAMILIES)
def test_kernel_solves_the_real_normal_equations(cases, gpu_states, gpu_gn, name, step, precision):
    case = cases(name)
    pk, opts = _prepare(case)
    obs, vis, x = gpu_states(case, name)
    out = gpu_linearize(pk, opts, obs, vis, x, step, precision)
    holder = lib.DescHolder(pk)
    st = check_real_systems(gpu_gn, zip(out['A'], out['g']), holder.desc, precision)
    print(name, step, precision, _maxima(st))


@pytest.mark.gpu
@pytest.mark.parametrize('precision', ['f32', 'f64'])
def test_kernel_rank_deficient_frames_are_flagged_and_recovered(cases, precision):
    """The product kernel's not-positive-definite exit (see test_emu_parity.py for the host build): a first frame seen
    through one marker and a second through two leave the root orientation unobserved, the Cholesky gives up, the frame
    takes the Cauchy step and is flagged MOSH2_ST_GN_FALLBACK; the later frames are not, and the solution comes back to the
    float64 oracle's once all markers are seen."""
    from conftest import dense_obs
    from moshpp_b200.mocap_interface import MocapSession
    from oracle import stageii
    case = cases('C1')
    obs, vis = dense_obs(case)
    vis = vis.copy()
    vis[0, 1:] = False
    vis[1, 2:] = False
    res = gpu_solve(case, precision=precision, obs_vis=(obs, vis))
    assert (res.status[:2] & lib.ST_GN_FALLBACK).all() and not (res.status[2:] & lib.ST_GN_FALLBACK).any()
    assert (res.status & lib.ST_SOLVED).all() and np.isfinite(res.pose).all() and np.isfinite(res.errs).all()
    mocap = MocapSession(case['mocap_fname'], case['cfg'].mocap.unit)
    col = {l: i for i, l in enumerate(mocap.labels)}
    for f, keep in ((0, 1), (1, 2)):
        for l in case['latent_labels'][keep:]:
            mocap.markers[f, col[l]] = 0.0
    ref = stageii.mosh_stageii(case['mocap_fname'], case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'],
                               case['marker_meta'], mocap=mocap)
    d = np.abs(res.pose - ref['_pose_reduced']).max(1)
    sse = ref['stageii_debug_details']['stageii_errs']['data']
    assert d[-1] < 0.1 * d[2] or d[-1] < 1e-2
    assert np.abs(res.errs[-3:, 0] / sse[-3:] - 1).max() < 0.05
