"""Stage I's device half against float64, for every body family and in each workspace layout it runs in.

Stage I linearises every picked frame with the Stage-II kernel in linearise mode (``mosh2_job_linearize``, float64 through
``stagei.DeviceBackend``), in a mode Stage II never uses: the shape directions are the linear block, ``jd_lin`` makes those
columns move the joints, and they are free in Step 1 as well as in Step 2.  A solve hides a wrong Jacobian (the dog-leg's
rho uses the true SSE), so this module compares the linearisation itself, at given states:

  * one linearisation per frame (J, r, vp, markers_sim, A, g and the SSE columns) against a float64 reference built here
    from oracle.lbs (posed attachment vertices and their pose and shape derivatives), oracle.markers (simulated markers and
    their local derivatives) and the oracle's prior terms -- the device's shape column is the derivative at FIXED attachment
    coefficients, the oracle's data column (oracle/stagei.py) without its Fp dk/dbetas term, which the host adds;
  * the block-arrow normal equations ``StageI.evaluate`` assembles (rows and columns: betas | latent markers | frames)
    against J^T J and -J^T r of ``oracle.stagei.StageISolver.residual`` at the same unknowns: the chain through dk/dbetas,
    the init, surface and shape-prior terms and the point-to-mesh distance;
  * the float64 workspace layouts with a linear block: shared memory with 20- and 10-marker tiles and the global workspace
    (the plan of every case is pinned below), and on MANO the launch switches of the kernel;
  * ``mosh_stagei`` end to end against ``oracle.mosh_stagei`` for the families test_stagei.py does not run.

States: random shape, root, body and hand poses and translations; observations the latent markers moved rigidly with the
root plus 2 cm noise; frame 1 with three markers hidden.  Every GPU test has a CPU twin on the host build of the device
source (``EmuStageIBackend``), which sets the bounds: the library linearises in float64, so they are summation order only.
Measures, per frame (as tests/test_gpu_normal_equations.py):
  J     |J - J_ref| / max |J_ref[:, col]| per column; rows of hidden markers exactly zero
  r     |r - r_ref| / wt_data (metres), vp / markers |. - ref| (metres)
  A     |A_ij - A_ref_ij| / sqrt(A_ref_ii A_ref_jj)
  g     |g - g_ref| / (sqrt(A_ref_ii) |r_all|), r_all the residual of all terms
  SSE   relative to the float64 value; the data SSE relative to 2 |r_data| (wt_data sqrt(3 n_vis))
"""
import numpy as np
import pytest

from conftest import EmuStageIBackend, stagei_case
from moshpp_b200 import lib
from moshpp_b200 import stagei as product
from oracle import mesh_distance as omd
from oracle import stagei as oracle
from oracle.lbs import LBS
from oracle.markers import TransformedCoeffs, transformed_lms
from oracle.prior import HORSE_JANGLES_IDS, HORSE_JANGLES_SIGNS, horse_joint_angles
from oracle.rigid import rodrigues
from test_face_reference_size import _NoBackend, _relayout, emu_plan  # noqa: F401 (emu_plan: a fixture)
from test_gpu_normal_equations import COL
from test_stagei import _compare

# name: (configuration, make_case arguments, marker count of a relayout (test_face_reference_size.LAYOUTS) or None)
CASES = {
    'C1': ('C1', {}, None), 'C1-65': ('C1', {}, 65), 'C1-90': ('C1', {}, 90),
    'C2': ('C2', {}, None),
    'C3': ('C3', {}, None),
    'C4L': ('C4', {}, None), 'C4R': ('C4', dict(hand_side='right'), None), 'C4L-65': ('C4', {}, 65), 'C4L-90': ('C4', {}, 90),
    'CH': ('CH', {}, None),
}
# the float64 workspace plan of each case (markers per tile, global workspace): mosh2_host::plan_workspace
PLAN = {'C1': (10, 0), 'C1-65': (10, 1), 'C1-90': (10, 1), 'C2': (10, 1), 'C3': (10, 1),
        'C4L': (20, 0), 'C4R': (20, 0), 'C4L-65': (20, 0), 'C4L-90': (10, 1), 'CH': (10, 1)}
SWITCHED = 'C4L'         # the shared-memory family the launch switches run on
SWITCHES = [('MOSH2_DEV_TILE', '10'), ('MOSH2_DEV_BIG', '1'), ('MOSH2_DEV_NO_TC', '1'), ('MOSH2_DEV_THREADS', '256'),
            ('MOSH2_DEV_THREADS', '128')]
ANNEAL = {1: 0.5, 2: 0.25}       # an annealing factor of each step (Step 1 runs at 1 and 1/2, Step 2 at 1/4 and 1/8)
N_FRAMES = 3
HIDDEN = (1, (0, 5, -1))         # frame, markers
# float64: summation order only
F64 = dict(J=1e-10, r=1e-12, vp=1e-12, markers=1e-12, A=1e-10, g=1e-10, sse=1e-10, data=1e-12)
ARROW = dict(A=1e-10, g=1e-10)


# ---- the problem at a given state -------------------------------------------------------------------------------------

def _problem(cases, name, backend, seed=11):
    """A StageI of ``name`` at a random state, and the oracle's StageISolver of the same frames at the same state."""
    config, kw, n_markers = CASES[name]
    case, cfg, _ = stagei_case(cases, config, 1, **kw)
    meta = case['marker_meta'] if n_markers is None else _relayout(case, n_markers)[1]
    labels = list(meta['marker_vids'])
    blank = [{l: np.zeros(3) for l in labels} for _ in range(N_FRAMES)]
    s = product.StageI(blank, cfg, meta, backend=backend)
    assert s.free_betas and s.nb == 16 and s.M == len(labels)
    rng = np.random.default_rng(seed)
    F, P = s.F, s.pose.shape[1]
    s.betas[:s.nb] = rng.normal(0, 1.0, s.nb)
    s.pose[:, :3] = rng.normal(0, 1.0, (F, 3))
    s.pose[:, 3:] = rng.normal(0, 0.2, (F, P - 3))
    s.trans[:] = rng.normal(0, 0.3, (F, 3))
    frames = []
    for f in range(F):
        obs = s.ml.dot(rodrigues(s.pose[f, :3]).T) + s.trans[f] + rng.normal(0, 0.02, s.ml.shape)
        frames.append({l: obs[i] for i, l in enumerate(labels)})
    f, hide = HIDDEN
    for i in hide:
        del frames[f][labels[i]]
    s.obs[:], s.vis[:] = 0.0, False
    for f, fr in enumerate(frames):
        for i, l in enumerate(labels):
            if l in fr:
                s.obs[f, i], s.vis[f, i] = fr[l], True
    assert s.vis.sum() == F * s.M - len(hide)
    o = oracle.StageISolver(frames, cfg, meta)
    o.betas[:], o.ml, o.pose[:], o.trans[:] = s.betas, s.ml.copy(), s.pose, s.trans
    return s, o


def _evaluate(cases, name, backend, step):
    """``StageI.evaluate`` with the normal equations at the state of ``_problem``: (s, o, weights, dev, A, g, pk, free, n_p)."""
    s, o = _problem(cases, name, backend)
    wts = s.weights_for(ANNEAL[step])
    _, _, dev, A, g, (pk, free, n_p) = s.evaluate(True, wts, step == 2)
    assert pk.n_dmpl == s.nb and len(free) == n_p + s.nb
    assert list(free[n_p:]) == [3 + pk.p_red + i for i in range(s.nb)]          # the shape columns are free in both steps
    return s, o, wts, dev, A, g, pk, free, n_p


# ---- 1. one linearisation per frame -----------------------------------------------------------------------------------

def frame_reference(s, o, wts, free, f, detailed):
    """Float64 rows of frame ``f`` in the device's columns ``free`` (x = [trans | pose | betas[:nb]]): data at wt_data, the
    body prior at wt_poseB (max-mixture component chosen in float64), the horse's joint angles at 2 wt_poseB and, in Step 2,
    the fingers at wt_poseH.  Returns J, r (data rows, zero where hidden), vp, markers, A, g, r_all and the SSE per column of
    mosh2_lin_out.errs (the kernel reports the horse's joint-angle term in the poseH column)."""
    M, nb, P = s.M, s.nb, o.model.pose_size
    n = len(free)
    col = {int(i): c for c, i in enumerate(free)}
    tc = TransformedCoeffs(o.can_v(), s.ml)
    tri = tc.closest[:, :3]
    verts, dv_pose, dv_beta = LBS(o.model, tri.reshape(-1))(s.pose[f], o.betas, s.trans[f], True, beta_ids=np.arange(nb))
    v = verts.reshape(M, 3, 3)
    sim, loc = transformed_lms(tc, v[:, 0], v[:, 1], v[:, 2], True)
    dsim = np.concatenate([np.broadcast_to(np.eye(3), (M, 3, 3)),                         # d sim / d [trans | pose | betas]
                           np.einsum('mik,mkp->mip', loc, dv_pose.reshape(M, 9, P)),
                           np.einsum('mik,mkb->mib', loc, dv_beta.reshape(M, 9, nb))], axis=2)
    w = wts['data'] * s.vis[f]
    J = (w[:, None, None] * dsim[:, :, free]).reshape(3 * M, n)
    r = (w[:, None] * (sim - s.obs[f])).reshape(-1)
    rows, sse = [(r, J)], np.zeros(len(lib.ERR_NAMES))
    sse[COL['data']] = (r ** 2).sum()

    def add(term, rr, dr, pids):
        Jt = np.zeros((len(rr), n))
        for k, pid in enumerate(pids):
            if 3 + pid in col:
                Jt[:, col[3 + pid]] = dr[:, k]
        rows.append((rr, Jt))
        sse[COL[term]] += (rr ** 2).sum()

    if len(o.body_ids) and o.prior is not None:
        xb = s.pose[f, o.body_ids]
        add('poseB', o.prior.r(xb) * wts['poseB'], o.prior.dr_wrt_x(xb) * wts['poseB'], o.body_ids)
        if o.model.model_type == 'animal_horse':
            ra = horse_joint_angles(xb) * 2.0 * wts['poseB']
            add('poseH', ra, np.diag(2.0 * HORSE_JANGLES_SIGNS * ra), np.asarray(o.body_ids)[HORSE_JANGLES_IDS])
    if detailed and o.optimize_fingers:
        add('poseH', s.pose[f, o.finger_ids] * wts['poseH'], np.eye(len(o.finger_ids)) * wts['poseH'], o.finger_ids)
    r_all = np.concatenate([a for a, _ in rows])
    J_all = np.vstack([b for _, b in rows])
    return dict(J=J, r=r, vp=verts, markers=sim, A=J_all.T @ J_all, g=-J_all.T @ r_all, r_all=r_all, sse=sse,
                n_vis=int(s.vis[f].sum()))


def linearisation_errors(s, o, wts, dev, pk, free, detailed):
    """Compares every frame of ``dev`` (backend.linearize, build = 1) with ``frame_reference`` and asserts ``F64``."""
    ids = o.pose_ids_for(detailed)
    assert pk.p_red == o.model.pose_size and [int(i) - 3 for i in free[3:3 + len(ids)]] == list(ids)
    assert np.abs(s.can(s.betas[:s.nb]) - o.can_v()).max() < 1e-12
    assert np.array_equal(pk.closest, TransformedCoeffs(o.can_v(), s.ml).closest[:, :3]), 'attachment triangles'
    st = {k: 0.0 for k in F64}
    for f in range(s.F):
        ref = frame_reference(s, o, wts, free, f, detailed)
        hidden = np.repeat(~s.vis[f], 3)
        assert not np.any(dev['J'][f][hidden]) and not np.any(dev['r'][f][hidden]), f
        e = {}
        e['J'] = (np.abs(dev['J'][f] - ref['J']) / np.maximum(np.abs(ref['J']).max(0), 1e-300)).max()
        e['r'] = np.abs(dev['r'][f] - ref['r']).max() / wts['data']
        e['vp'] = np.abs(dev['vp'][f] - ref['vp']).max()
        e['markers'] = np.abs(dev['markers_sim'][f] - ref['markers']).max()
        d = np.sqrt(np.diag(ref['A']))
        assert np.all(d > 0)
        e['A'] = (np.abs(dev['A'][f] - ref['A']) / np.outer(d, d)).max()
        e['g'] = (np.abs(dev['g'][f] - ref['g']) / (d * np.linalg.norm(ref['r_all']))).max()
        got, want = dev['errs'][f], ref['sse']
        assert np.array_equal(got == 0, want == 0), (f, got, want)
        c0 = COL['data']
        e['data'] = abs(got[c0] - want[c0]) / (2 * np.sqrt(want[c0]) * wts['data'] * np.sqrt(3 * ref['n_vis']))
        e['sse'] = max([abs(got[c] - want[c]) / want[c] for c in range(len(want)) if c != c0 and want[c]] + [0.0])
        for k, val in e.items():
            assert val <= F64[k], (f, k, val, F64[k])
            st[k] = max(st[k], float(val))
    return st


def _check_linearisation(cases, name, backend, step):
    s, o, wts, dev, _, _, pk, free, _ = _evaluate(cases, name, backend, step)
    st = linearisation_errors(s, o, wts, dev, pk, free, step == 2)
    print(name, step, {k: float('%.2g' % v) for k, v in st.items()})


@pytest.mark.parametrize('step', [1, 2])
@pytest.mark.parametrize('name', list(CASES))
def test_device_source_stagei_linearisation_equals_float64(cases, name, step):
    _check_linearisation(cases, name, EmuStageIBackend(), step)


@pytest.mark.gpu
@pytest.mark.parametrize('step', [1, 2])
@pytest.mark.parametrize('name', list(CASES))
def test_kernel_stagei_linearisation_equals_float64(cases, name, step):
    _check_linearisation(cases, name, product.DeviceBackend(), step)


# ---- 2. the block-arrow normal equations ------------------------------------------------------------------------------

def arrow_errors(s, o, A, g, free, n_p, detailed):
    """``StageI.evaluate``'s A and g against the oracle's J^T J and -J^T r (oracle/dogleg.py) at the same unknowns."""
    pose_ids = o.pose_ids_for(detailed)
    assert [int(i) - 3 for i in free[3:n_p]] == list(pose_ids)
    r, J = o.residual(o.get_x(pose_ids, True), True, pose_ids, True, o.weights_for(ANNEAL[2 if detailed else 1]), detailed)
    A_ref, g_ref = J.T @ J, -J.T @ r
    assert A.shape == A_ref.shape
    d = np.sqrt(np.diag(A_ref))
    assert np.all(d > 0)
    st = dict(A=(np.abs(A - A_ref) / np.outer(d, d)).max(), g=(np.abs(g - g_ref) / (d * np.linalg.norm(r))).max())
    for k, v in st.items():
        assert v <= ARROW[k], (k, v)
    return st


def _nearest_parts(faces, tri, part):
    """The vertex ids of each nearest part: a triangle (part 0), an edge (1-3) or a vertex (4-6).  An edge or a vertex is
    shared by several triangles, and which of them a search reports is a tie."""
    out = []
    for t, p in zip(tri, part):
        fv = faces[t]
        out.append(tuple(sorted(fv if p == 0 else (fv[p - 1], fv[p % 3]) if p <= 3 else (fv[p - 4],))))
    return out


def _check_arrow(cases, name, backend, step):
    s, o, _, _, A, g, _, free, n_p = _evaluate(cases, name, backend, step)
    # the nearest part of the mesh to every latent marker: the float64 brute force's (the closed forms are float64)
    can_v = s.can(s.betas[:s.nb])
    _, tri, part, _, _ = s.backend.squared_distance(s.ml, can_v, s.faces)
    _, _, _, tri_ref, part_ref = omd.somedistance(s.ml, o.can_v(), o.faces, kind=omd.KIND_SQUARED)
    assert _nearest_parts(s.faces, tri, part) == _nearest_parts(o.faces, tri_ref, part_ref)
    st = arrow_errors(s, o, A, g, free, n_p, step == 2)
    print(name, step, {k: float('%.2g' % v) for k, v in st.items()})


@pytest.mark.parametrize('step', [1, 2])
@pytest.mark.parametrize('name', list(CASES))
def test_device_source_stagei_normal_equations_equal_oracle(cases, name, step):
    _check_arrow(cases, name, EmuStageIBackend(), step)


@pytest.mark.gpu
@pytest.mark.parametrize('step', [1, 2])
@pytest.mark.parametrize('name', list(CASES))
def test_kernel_stagei_normal_equations_equal_oracle(cases, name, step):
    _check_arrow(cases, name, product.DeviceBackend(), step)


# ---- 3. layouts -------------------------------------------------------------------------------------------------------

def test_cases_cover_the_float64_layouts_with_a_linear_block(cases, emu_plan):
    """The float64 plan of every case above: together they run shared memory with 20- and with 10-marker tiles and the
    global workspace, each with the shape directions as linear block (n_dmpl > 0; the joint directions c_jd staged in shared
    memory except in the global workspace).  A planner change that moves a case fails here: re-pin PLAN and keep the
    three layouts covered."""
    got = {}
    for name in CASES:
        s, _ = _problem(cases, name, _NoBackend())
        pk = s.pack_for(True)
        assert pk.n_dmpl == 16
        p = emu_plan(pk, 'f64', 0)
        assert p['smem'] <= p['budget'], (name, p)
        got[name] = (p['tile'], p['big'])
    assert got == PLAN
    assert set(PLAN.values()) == {(20, 0), (10, 0), (10, 1)}


@pytest.mark.gpu
@pytest.mark.parametrize('switch', SWITCHES)
@pytest.mark.parametrize('step', [1, 2])
def test_kernel_stagei_linearisation_under_other_launch_layouts(cases, step, switch, monkeypatch):
    """MANO's shared 20-marker tiles with 10-marker tiles, the global workspace, J^T J on the CUDA cores instead of DMMA, and
    256 or 128 threads; the same bounds.  The tile, workspace and tensor-core switches are read when the job is created, the
    thread count at every launch: both happen inside ``linearize``."""
    monkeypatch.setenv(*switch)
    s, o, wts, dev, _, _, pk, free, _ = _evaluate(cases, SWITCHED, product.DeviceBackend(), step)
    monkeypatch.delenv(switch[0])
    st = linearisation_errors(s, o, wts, dev, pk, free, step == 2)
    print(SWITCHED, step, switch, {k: float('%.2g' % v) for k, v in st.items()})


# ---- 4. end to end ----------------------------------------------------------------------------------------------------

END_TO_END = {'C1': ('C1', {}), 'C3': ('C3', {}), 'C4': ('C4', {}), 'CH': ('CH', {})}
MAXITER = 3


def _end_to_end(cases, name, backend, tol):
    config, kw = END_TO_END[name]
    case, cfg, frames = stagei_case(cases, config, 4, **kw)
    cfg.opt_settings.maxiter = MAXITER
    ref = oracle.mosh_stagei(frames, cfg, marker_meta=case['marker_meta'])
    out = product.mosh_stagei(frames, cfg, marker_meta=case['marker_meta'], backend=backend)
    _compare(out, ref, tol)
    st, rs = out['stagei_debug_details']['b200'], ref['stagei_debug_details']['oracle_stats']
    print(name, st, rs)
    assert st['linearisations'] == rs['j_evals'] and st['iterations'] == rs['iterations'] and st['minimisations'] == 4
    assert np.abs(out['betas'][:cfg.surface_model.num_betas]).max() > 1e-3


@pytest.mark.parametrize('name', list(END_TO_END))
def test_block_solve_on_device_source_equals_oracle(cases, name):
    _end_to_end(cases, name, EmuStageIBackend(), 1e-9)


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(END_TO_END))
def test_stagei_on_the_gpu_equals_oracle(cases, name):
    _end_to_end(cases, name, None, 1e-6)


@pytest.mark.gpu
def test_given_betas_are_kept_on_the_gpu(cases, tmp_path):
    """optimize_betas off with a betas file (chmosh.py:92-97,169-172) through the CUDA library: the shape stays, the latent
    markers and poses agree with the oracle."""
    case, cfg, frames = stagei_case(cases, 'C1', 3)
    cfg.moshpp.optimize_betas = False
    fn = str(tmp_path / 'betas.npz')
    np.savez(fn, betas=case['betas'])
    ref = oracle.mosh_stagei(frames, cfg, betas_fname=fn, marker_meta=case['marker_meta'])
    out = product.mosh_stagei(frames, cfg, betas_fname=fn, marker_meta=case['marker_meta'])
    _compare(out, ref, 1e-6)
    nb = cfg.surface_model.num_betas
    assert np.array_equal(out['betas'][:nb], case['betas'][:nb]) and 'beta' not in out['stagei_debug_details']['stagei_errs']
