"""Stage II's joint minimisation of the sequence objective (``sequence_sweeps``; DESIGN.md section 11).

S = sum_k E_k(x_k) + sum_{k>=2} |w (p_k - 2 p_{k-1} + p_{k-2})|^2 + [DMPL] sum_{k>=1} |6 (d_k - d_{k-1})|^2 over the processed
frames of a capture, minimised from the causal solve by three-colour block Gauss-Seidel sweeps of the reference's Step-2 dog-leg.
The float64 oracle below restates the sweeps on the unchanged ``oracle.stageii`` solver, with the temporal residuals kept as
residuals.  The host build of the device source (tests/emu/mosh2_emu_sequence.cpp) is checked against it; the GPU tests run
the CUDA sweeps.
"""
from __future__ import annotations

import ctypes as C
import functools
import json
import os
import pickle
import shutil

import numpy as np
import pytest

from conftest import EmuStageIBackend, dense_obs, run_oracle
from moshpp_b200 import build, chmosh, lib, mosh_head, stagei, synth
from oracle import stageii as oracle_stageii

TOL_EXACT = chmosh.BOUNDARY_TOL['exact']


# ---- float64 oracle of the sweeps ----------------------------------------------------------------------------------------------
class _SeqObjective(oracle_stageii._Objective):
    """A frame's Step-2 objective plus the temporal residuals that contain it: ``velo`` rows wv (a p + b) over the whole reduced
    pose, ``dm`` rows wx (a d + b) over the DMPL coefficients (a: the frame's coefficient, b: the neighbours' part)."""

    def __init__(self, solver, obs, vis, terms, pose_ids, free_dmpl, velo, dm, wv, wx):
        super().__init__(solver, obs, vis, terms, pose_ids, free_dmpl)
        self.velo, self.dm, self.wv, self.wx = velo, dm, wv, wx

    def _temporal(self, want_jac):
        s, npi = self.s, len(self.pose_ids)
        rs, Js = [], []
        for a, b in self.velo:
            rs.append(self.wv * (a * s.pose + b))
            if want_jac:
                J = np.zeros((len(s.pose), self.n))
                J[self.pose_ids, 3 + np.arange(npi)] = self.wv * a
                Js.append(J)
        for a, b in self.dm:
            rs.append(self.wx * (a * s.betas[s.dmpl_ids] + b))
            if want_jac:
                J = np.zeros((s.n_dm, self.n))
                J[:, 3 + npi:3 + npi + s.n_dm] = np.eye(s.n_dm) * self.wx * a
                Js.append(J)
        return rs, Js

    def __call__(self, x, want_jac):
        out = super().__call__(x, want_jac)
        rs, Js = self._temporal(want_jac)
        if want_jac:
            r, J = out
            return np.concatenate([r] + rs), np.vstack([J] + Js)
        return np.concatenate([out] + rs)


def temporal_rows(P, D, k, n, dyn):
    """(a, b) of every residual that contains frame k, given the rows P (pose) and D (DMPL) of the n processed frames."""
    velo, dm = [], []
    if k >= 2:
        velo.append((1.0, P[k - 2] - 2.0 * P[k - 1]))
    if 1 <= k <= n - 2:
        velo.append((-2.0, P[k - 1] + P[k + 1]))
    if k <= n - 3:
        velo.append((1.0, P[k + 2] - 2.0 * P[k + 1]))
    if dyn:
        if k >= 1:
            dm.append((1.0, -D[k - 1]))
        if k <= n - 2:
            dm.append((-1.0, D[k + 1]))
    return velo, dm


def oracle_sequence(case, max_sweeps, tol=TOL_EXACT, obs_vis=None, on_colour=None):
    """The causal oracle, then at most ``max_sweeps`` sweeps.  Returns (causal output, final rows P, T, L (linear block),
    sweeps, per-sweep deltas, per-frame Jacobian builds of the sweeps, S causal, S final)."""
    cfg = case['cfg']
    obs, vis = obs_vis if obs_vis is not None else dense_obs(case)
    out = run_oracle(case, mocap=_Mocap(case, obs, vis))
    s = oracle_stageii.StageIISolver(cfg, case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])
    frames = [None if not v.any() else (np.flatnonzero(v), o[v]) for o, v in zip(obs, vis)]
    proc = [f for f, fr in enumerate(frames) if fr is not None]
    assert np.array_equal(out['stageii_debug_details']['frame_ids'], proc)
    n = len(proc)
    P = out['_pose_reduced'].copy()
    T = out['trans'].copy()
    L = np.zeros((n, s.nd))
    if s.optimize_dynamics:
        L[:, :s.n_dm] = out['dmpls']
    if len(s.expr_ids):
        L[:, s.n_dm:] = out['expression'][:, :len(s.expr_ids)]
    dyn = s.optimize_dynamics
    wv, wx = float(s.wts['stageii_wt_velo']), 6.0
    nbody = min(int(case['pack'].body_dof), 66)

    def frame_e(k):
        vis_k, obs_k = frames[proc[k]]
        s.pose[:] = P[k]; s.trans[:] = T[k]
        if s.nd:
            s.betas[s.lin_ids] = L[k]
        terms, _ = s.frame_terms(len(vis_k))
        return sum(oracle_stageii._Objective(s, obs_k, vis_k, terms, s.step2_ids, s.nd > 0).term_sse().values())

    def objective(E):
        velo, extrap = chmosh.sequence_temporal_sse(P, L[:, :s.n_dm] if dyn else None, wv, wx, s.n_dm if dyn else 0)
        return float(E.sum() + velo.sum() + extrap.sum())

    E = np.array([frame_e(k) for k in range(n)])
    s_causal = objective(E)
    builds = np.zeros(n, dtype=np.int64)
    deltas, sweeps = [], 0
    while sweeps < max_sweeps:
        md = np.zeros(4)
        for c in range(3):
            for k in range(c, n, 3):
                vis_k, obs_k = frames[proc[k]]
                s.pose[:] = P[k]; s.trans[:] = T[k]
                if s.nd:
                    s.betas[s.lin_ids] = L[k]
                terms, _ = s.frame_terms(len(vis_k))
                velo, dm = temporal_rows(P, L[:, :s.n_dm], k, n, dyn)
                obj = _SeqObjective(s, obs_k, vis_k, terms, s.step2_ids, s.nd > 0, velo, dm, wv, wx)
                j0 = s.stats['j_evals']
                s._minimize(obj, 1e-2)
                builds[k] += s.stats['j_evals'] - j0
                dp = np.abs(s.pose - P[k])
                md[0] = max(md[0], dp[:nbody].max())
                md[1] = max(md[1], dp[nbody:].max() if len(dp) > nbody else 0.0)
                md[2] = max(md[2], np.abs(s.trans - T[k]).max())
                if s.nd:
                    md[3] = max(md[3], np.abs(s.betas[s.lin_ids] - L[k]).max())
                    L[k] = s.betas[s.lin_ids]
                P[k] = s.pose; T[k] = s.trans
                E[k] = sum(obj.term_sse().values())
            if on_colour is not None:
                on_colour(objective(E))
        deltas.append(md)
        sweeps += 1
        if (md <= np.asarray(tol)).all():
            break
    return dict(out=out, P=P, T=T, L=L, sweeps=sweeps, deltas=deltas, builds=builds, S_causal=s_causal, S=objective(E), proc=proc)


class _Mocap:
    """The oracle's mocap argument for a capture given as dense observations in latent-label order (metres)."""

    def __init__(self, case, obs, vis):
        self.markers = np.where(vis[..., None], obs, 0.0)
        self.labels = list(case['latent_labels'])
        self.frame_rate = 120.0

    def __len__(self):
        return len(self.markers)

    def time_length(self):
        return len(self.markers) / self.frame_rate


# ---- host build ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def emu_handle():
    return C.CDLL(build.build_emu())


def case_options(case):
    pk, cfg = case['pack'], case['cfg']
    return lib.make_options(cfg.opt_settings.weights, optimize_fingers=bool(cfg.moshpp.optimize_fingers) and pk.finger_hi > pk.finger_lo,
                            optimize_dynamics=bool(cfg.moshpp.optimize_dynamics),
                            optimize_face=bool(cfg.moshpp.optimize_face) and pk.n_expr > 0)


def emu_sequence(handle, case, obs, vis, max_sweeps, counts=None, tol=TOL_EXACT, precision=lib.MOSH2_F64):
    pk = case['pack']
    h = lib.DescHolder(pk)
    opt = case_options(case)
    counts = np.ascontiguousarray(counts if counts is not None else [len(obs)], dtype=np.int32)
    res = lib.ResultArrays(len(obs), lib.pack_dims(pk))
    o = np.ascontiguousarray(obs, dtype=np.float64)
    v8 = np.ascontiguousarray(vis, dtype=np.uint8)
    sched = lib.make_schedule(0, 0)
    t = np.ascontiguousarray(tol, dtype=np.float64)
    sweeps = C.c_int32()
    deltas = np.zeros((max(max_sweeps, 1), 4))
    rc = handle.mosh2_emu_solve_sequence(C.byref(h.desc), C.byref(opt), len(counts), counts.ctypes.data_as(lib._i32p),
                                         o.ctypes.data_as(lib._f64p), v8.ctypes.data_as(lib._u8p), C.byref(sched), precision,
                                         max_sweeps, t.ctypes.data_as(lib._f64p), C.byref(res.c), C.byref(sweeps),
                                         deltas.ctypes.data_as(lib._f64p))
    assert rc == 0
    return res, sweeps.value, deltas[:sweeps.value]


def with_dropout(case, lo, hi):
    """The case's capture with every marker of frames [lo, hi) missing (frames the reference skips)."""
    obs, vis = dense_obs(case)
    vis = vis.copy()
    vis[lo:hi] = False
    return obs, vis


CASES = {'C1': None, 'C2': (6, 8), 'C3': (4, 5), 'CF': None, 'C4': None}


@pytest.mark.parametrize('name', list(CASES))
def test_oracle_sweeps_lower_the_sequence_objective(cases, name):
    """S never rises from one colour launch to the next, and the sweeps end below the causal S."""
    case = cases(name)
    obs_vis = with_dropout(case, *CASES[name]) if CASES[name] else None
    trace = []
    r = oracle_sequence(case, 3, obs_vis=obs_vis, on_colour=trace.append)
    seq = [r['S_causal']] + trace
    assert all(b <= a * (1 + 1e-12) for a, b in zip(seq, seq[1:])), seq
    assert r['S'] < r['S_causal']


@pytest.mark.parametrize('name', list(CASES))
def test_device_source_sweeps_equal_the_oracle(cases, emu_handle, name):
    """The host build's sweeps equal the oracle's in float64: rows to 1e-9, the same sweep count, the same Jacobian builds per
    frame; skipped frames stay skipped and their neighbours are the processed frames around them."""
    case = cases(name)
    obs, vis = with_dropout(case, *CASES[name]) if CASES[name] else dense_obs(case)
    r = oracle_sequence(case, 4, obs_vis=(obs, vis))
    causal, _, _ = emu_sequence(emu_handle, case, obs, vis, 0)
    causal_builds = causal.counters[:, 2].copy()
    res, sweeps, deltas = emu_sequence(emu_handle, case, obs, vis, 4)
    fid = np.flatnonzero(res.status & lib.ST_SOLVED)
    assert np.array_equal(fid, r['proc'])
    assert sweeps == r['sweeps']
    assert np.abs(res.pose[fid] - r['P']).max() < 1e-9
    assert np.abs(res.trans[fid] - r['T']).max() < 1e-9
    if r['L'].shape[1]:
        assert np.abs(res.dmpls[fid] - r['L']).max() < 1e-9
    pk = case['pack']
    if name == 'C3':                 # the DMPL case: the DMPL differences take part and the coefficients move in the sweeps
        assert bool(case['cfg'].moshpp.optimize_dynamics) and pk.n_dmpl - pk.n_expr > 0
        assert np.abs(res.dmpls[fid, :pk.n_dmpl - pk.n_expr] - causal.dmpls[fid, :pk.n_dmpl - pk.n_expr]).max() > 1e-6
    assert np.array_equal(res.counters[fid, 2] - causal_builds[fid], r['builds'])
    assert np.allclose(deltas, np.array(r['deltas']), rtol=1e-6, atol=1e-12)


def _joint_residual(case, obs_vis, x_rows):
    """The whole sequence objective of a tiny capture as one least-squares problem over every processed frame's Step-2 variables
    (``x_rows`` [F', 3 + P_red + n_lin]): r(x) and its Jacobian, from the oracle's frame objectives and the temporal rows."""
    obs, vis = obs_vis
    s = oracle_stageii.StageIISolver(case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])
    proc = [f for f in range(len(obs)) if vis[f].any()]
    n, PR, wv = len(proc), len(s.pose), float(s.wts['stageii_wt_velo'])
    ids = np.asarray(s.step2_ids)
    nfree = 3 + len(ids) + s.nd

    def unpack(z):
        X = x_rows.copy()
        Z = z.reshape(n, nfree)
        X[:, :3] = Z[:, :3]
        X[:, 3 + ids] = Z[:, 3:3 + len(ids)]
        if s.nd:
            X[:, 3 + PR:] = Z[:, 3 + len(ids):]
        return X

    def fun(z):
        X = unpack(z)
        rows, blocks = [], []
        for k, f in enumerate(proc):
            v = np.flatnonzero(vis[f])
            s.trans[:] = X[k, :3]; s.pose[:] = X[k, 3:3 + PR]
            if s.nd:
                s.betas[s.lin_ids] = X[k, 3 + PR:]
            terms, _ = s.frame_terms(len(v))
            obj = oracle_stageii._Objective(s, obs[f][v], v, terms, s.step2_ids, s.nd > 0)
            r, J = obj(obj.x0(), True)
            rows.append(r)
            blocks.append((k, J))
        nr = sum(len(r) for r in rows) + max(n - 2, 0) * PR
        J = np.zeros((nr, n * nfree))
        o = 0
        for (k, Jk), r in zip(blocks, rows):
            J[o:o + len(r), k * nfree:(k + 1) * nfree] = Jk
            o += len(r)
        P = X[:, 3:3 + PR]
        for k in range(2, n):
            rows.append(wv * (P[k] - 2 * P[k - 1] + P[k - 2]))
            for kk, a in ((k, 1.0), (k - 1, -2.0), (k - 2, 1.0)):
                J[o + ids, kk * nfree + 3 + np.arange(len(ids))] = wv * a
            o += PR
        return np.concatenate(rows), J

    def z_of(X):
        return np.concatenate([X[:, :3], X[:, 3 + ids], X[:, 3 + PR:]], axis=1).reshape(-1)
    return fun, z_of


def test_joint_optimum_is_nearer_the_sweeps_than_the_causal_solve(cases):
    """On a tiny capture, scipy's least_squares over every frame at once lowers S less from the swept result than from the causal
    one: the sweeps move towards the joint minimum.  (C1, first 6 frames; measured: S causal 2571.885, swept 2570.386; least_squares
    lowers S by 1.498 from the causal result and by 3.1e-8 from the swept one.)"""
    from scipy.optimize import least_squares
    case = cases('C1')
    obs, vis = dense_obs(case)
    obs, vis = obs[:6], vis[:6]
    r = oracle_sequence(case, 8, obs_vis=(obs, vis))
    causal = np.concatenate([r['out']['trans'], r['out']['_pose_reduced'], np.zeros((len(r['P']), r['L'].shape[1]))], axis=1)
    swept = np.concatenate([r['T'], r['P'], r['L']], axis=1)
    gains = {}
    for name, X in (('causal', causal), ('swept', swept)):
        fun, z_of = _joint_residual(case, (obs, vis), X)
        z0 = z_of(X)
        s0 = float((fun(z0)[0] ** 2).sum())
        sol = least_squares(lambda z: fun(z)[0], z0, jac=lambda z: fun(z)[1], method='lm', max_nfev=200, xtol=1e-14, ftol=1e-14)
        gains[name] = (s0, s0 - float((sol.fun ** 2).sum()))
    assert np.isclose(gains['causal'][0], r['S_causal'], rtol=1e-9) and np.isclose(gains['swept'][0], r['S'], rtol=1e-9)
    assert 0 <= gains['swept'][1] < gains['causal'][1]
    print('least_squares gain from causal / swept:', gains)


def test_two_capture_batch_equals_each_capture_alone(cases, emu_handle):
    case = cases('C2')
    obs, vis = dense_obs(case)
    a, b = 7, len(obs)
    both, sweeps_ab, _ = emu_sequence(emu_handle, case, obs, vis, 3, counts=[a, b - a])
    one, _, _ = emu_sequence(emu_handle, case, obs[:a], vis[:a], 3)
    two, _, _ = emu_sequence(emu_handle, case, obs[a:], vis[a:], 3)
    assert np.array_equal(both.pose[:a], one.pose) and np.array_equal(both.pose[a:], two.pose)
    assert np.array_equal(both.trans[:a], one.trans) and np.array_equal(both.trans[a:], two.trans)


# ---- plumbing ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('bad', [0, -1, 1.5, '2', True, [1]])
def test_bad_sweep_counts_raise(cases, bad):
    case = cases('C1')
    args = (case['mocap_fname'], case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])
    with pytest.raises(ValueError, match='sequence_sweeps'):
        chmosh.mosh_stageii(*args, sequence_sweeps=bad)
    with pytest.raises(ValueError, match='sequence_sweeps'):
        chmosh.mosh_stageii_batch([case['mocap_fname']], *args[1:], sequence_sweeps=bad)
    with pytest.raises(ValueError, match='sequence_sweeps'):
        chmosh.mosh_stageii_subjects([dict(cfg=case['cfg'], mocap_fnames=[case['mocap_fname']], markers_latent=case['markers_latent'],
                                           latent_labels=case['latent_labels'], betas=case['betas'], marker_meta=case['marker_meta'])],
                                     sequence_sweeps=bad)


def test_sweep_counts_that_are_accepted():
    assert chmosh.check_sequence_sweeps(None) is None
    assert chmosh.check_sequence_sweeps(1) == 1
    assert chmosh.check_sequence_sweeps(np.int64(7)) == 7


def test_temporal_sse_assigns_residuals_as_the_reference():
    rng = np.random.default_rng(0)
    P, D = rng.normal(size=(6, 5)), rng.normal(size=(6, 4))
    velo, extrap = chmosh.sequence_temporal_sse(P, D, 2.5, 6.0, 3)
    assert velo[:2].sum() == 0 and extrap[0] == 0
    assert np.isclose(velo[4], 6.25 * ((P[4] - 2 * P[3] + P[2]) ** 2).sum())
    assert np.isclose(extrap[3], 36.0 * ((D[3, :3] - D[2, :3]) ** 2).sum())


# ---- GPU ----------------------------------------------------------------------------------------------------------------------------
KEYS = ('pose', 'trans', 'dmpls', 'errs', 'status', 'counters')


def _gpu_sequence(case, obs, vis, max_sweeps, precision, tol=TOL_EXACT, dev_big=False):
    """Causal launch, then sweeps on one job, as ``chmosh.sequence_solve`` drives them.  ``dev_big``: the global-workspace layout
    forced (MOSH2_DEV_BIG)."""
    pk, opts, _ = chmosh.prepare_stageii(case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])
    old = os.environ.pop('MOSH2_DEV_BIG', None)
    if dev_big:
        os.environ['MOSH2_DEV_BIG'] = '1'
    model = lib.Model(pk, device=0)
    try:
        job = model.job([len(obs)], opts, chunk_len=0, chunk_warmup=0, precision=precision)
        try:
            job.upload(obs, vis)
            job.launch()
            r = job.download()
            causal = {k: None if getattr(r, k) is None else getattr(r, k).copy() for k in KEYS}
            sweeps = 0
            while sweeps < max_sweeps:
                md = job.sequence_sweep()
                sweeps += 1
                if (md <= np.asarray(tol)).all():
                    break
            r = job.download()
            return causal, {k: None if getattr(r, k) is None else getattr(r, k).copy() for k in KEYS}, sweeps
        finally:
            job.close()
    finally:
        model.close()
        os.environ.pop('MOSH2_DEV_BIG', None)
        if old is not None:
            os.environ['MOSH2_DEV_BIG'] = old


def _cuda_objective(case, res):
    """S of a CUDA result (chmosh.sequence_objective over the processed frames)."""
    pk, cfg = case['pack'], case['cfg']
    n_dm = pk.n_dmpl - pk.n_expr if cfg.moshpp.optimize_dynamics else 0
    fid = np.flatnonzero(res['status'] & lib.ST_SOLVED)
    w = cfg.opt_settings.weights
    return chmosh.sequence_objective(res['errs'][fid], res['pose'][fid], res['dmpls'][fid] if n_dm else None,
                                     float(w['stageii_wt_velo']), 6.0, n_dm)


@pytest.mark.gpu
@pytest.mark.parametrize('name,dev_big', [('C1', False), ('C2', False), ('C2', True), ('C3', False), ('CF', False)])
def test_f64_cuda_sweeps_equal_the_oracle(cases, name, dev_big):
    """float64: the CUDA sweeps equal the oracle's to the f64 parity bounds, and S of the CUDA result falls below the CUDA causal
    S.  C3 (SMPL-X + DMPL) and CF run the global-workspace layout in float64 by their size; C2 is also run with it forced."""
    case = cases(name)
    obs, vis = with_dropout(case, *CASES[name]) if CASES[name] else dense_obs(case)
    r = oracle_sequence(case, 4, obs_vis=(obs, vis))
    causal, res, sweeps = _gpu_sequence(case, obs, vis, 4, lib.MOSH2_F64, dev_big=dev_big)
    fid = np.flatnonzero(res['status'] & lib.ST_SOLVED)
    assert np.array_equal(fid, r['proc'])
    assert sweeps == r['sweeps']
    assert np.abs(res['pose'][fid] - r['P']).max() < 1e-8
    assert np.abs(res['trans'][fid] - r['T']).max() < 1e-8
    if r['L'].shape[1]:
        assert np.abs(res['dmpls'][fid] - r['L']).max() < 1e-8
    s_causal, s_joint = _cuda_objective(case, causal), _cuda_objective(case, res)
    assert s_joint < s_causal
    assert np.isclose(s_joint, r['S'], rtol=1e-7)


@pytest.mark.gpu
@pytest.mark.parametrize('name,dev_big', [('C1', False), ('C2', False), ('C2', True)])
def test_f32_cuda_sweeps_within_the_fast_mode_tolerances(cases, name, dev_big):
    """float32 (the fast preset's precision): three sweeps each against the oracle's three float64 sweeps, within BASELINE.md
    section 4's per-frame tolerances (1e-3 rad root + body, 1e-2 other pose coefficients, 1e-4 m); S of the result below the
    causal S."""
    case = cases(name)
    obs, vis = with_dropout(case, *CASES[name]) if CASES[name] else dense_obs(case)
    r = oracle_sequence(case, 3, tol=(0, 0, 0, 0), obs_vis=(obs, vis))
    causal, res, sweeps = _gpu_sequence(case, obs, vis, 3, lib.MOSH2_F32, tol=(0, 0, 0, 0), dev_big=dev_big)
    assert sweeps == r['sweeps'] == 3
    fid = np.flatnonzero(res['status'] & lib.ST_SOLVED)
    nb = min(case['pack'].body_dof, 66)
    assert np.abs(res['pose'][fid, :nb] - r['P'][:, :nb]).max() < 1e-3
    if r['P'].shape[1] > nb:
        assert np.abs(res['pose'][fid, nb:] - r['P'][:, nb:]).max() < 1e-2
    assert np.abs(res['trans'][fid] - r['T']).max() < 1e-4
    assert _cuda_objective(case, res) < _cuda_objective(case, causal)


def _args(case):
    return (case['mocap_fname'], case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])


def _equal(a, b, skip=('kernel_ms', 'wall_s', 'host_ms', 'subject_cache_hit')):
    if isinstance(a, dict):
        assert set(a) == set(b)
        for k in a:
            if k not in skip:
                _equal(a[k], b[k], skip)
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b)
        for x, y in zip(a, b):
            _equal(x, y, skip)
    elif isinstance(a, np.ndarray):
        assert a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a, b)
    else:
        assert a == b


@pytest.mark.gpu
def test_none_returns_the_causal_dictionary_bit_for_bit(cases):
    case = cases('C3')
    plain = chmosh.mosh_stageii(*_args(case))
    off = chmosh.mosh_stageii(*_args(case), sequence_sweeps=None)
    assert 'sequence_solve' not in off['stageii_debug_details']['b200']
    _equal(plain, off)
    on = chmosh.mosh_stageii(*_args(case), sequence_sweeps=8)
    rec = on['stageii_debug_details']['b200']['sequence_solve']
    assert set(rec) >= {'sweeps', 'converged', 'objective_causal', 'objective', 'max_delta'}
    assert rec['objective'] < rec['objective_causal']
    # the temporal columns are the reference's assignment of the joint solution's residuals
    b = on['stageii_debug_details']['b200']
    pose = b['pose_reduced']
    wv = float(case['cfg'].opt_settings.weights['stageii_wt_velo'])
    velo, extrap = chmosh.sequence_temporal_sse(pose, on['dmpls'], wv, 6.0, on['dmpls'].shape[1])
    assert np.allclose(on['stageii_debug_details']['stageii_errs']['velo'], velo[2:], rtol=1e-6, atol=1e-12)
    assert np.allclose(on['stageii_debug_details']['stageii_errs']['extrap_dmpl'], extrap[1:], rtol=1e-6, atol=1e-12)


@pytest.mark.gpu
def test_head_run_writes_the_sequence_solve_record(tmp_path):
    """The head, with Stage II bound to ``sequence_sweeps`` through functools.partial, writes the record into its pickle."""
    root = str(tmp_path)
    session = os.path.join(root, 'mocap', 'Synth DS', 'subject 01')
    os.makedirs(session)
    case = synth.make_case(os.path.join(root, 'models'), 'C2', frames=10, n_verts=1500)
    cap = os.path.join(session, 'take_00.npz')
    shutil.move(case['mocap_fname'], cap)
    with open(os.path.join(session, 'settings.json'), 'w') as f:
        json.dump({'gender': 'male'}, f)
    work = os.path.join(root, 'work')
    cfg = {'mocap.fname': cap, 'dirs.work_base_dir': work, 'dirs.support_base_dir': os.path.join(root, 'support'),
           'surface_model.type': 'smplh', 'surface_model.fname': case['cfg'].surface_model.fname,
           'moshpp.pose_body_prior_fname': case['cfg'].moshpp.pose_body_prior_fname,
           'moshpp.pose_hand_prior_fname': case['cfg'].moshpp.pose_hand_prior_fname, 'moshpp.optimize_fingers': True,
           'moshpp.stagei_frame_picker.num_frames': 4, 'moshpp.stagei_frame_picker.least_avail_markers': 0.8,
           'opt_settings.maxiter': 4, 'moshpp.head_marker_corr_fname': None}
    layout = os.path.join(work, 'SynthDS', 'SynthDS_smplh.json')
    os.makedirs(os.path.dirname(layout), exist_ok=True)
    stagei.write_marker_layout(layout, case['marker_meta'])
    np.random.seed(0)
    mp = mosh_head.run_moshpp_once(cfg, stagei_func=functools.partial(stagei.mosh_stagei, backend=EmuStageIBackend()),
                                   stageii_func=functools.partial(chmosh.mosh_stageii, sequence_sweeps=4))
    with open(mp.stageii_fname, 'rb') as f:
        s2 = pickle.load(f)
    rec = s2['stageii_debug_details']['b200']['sequence_solve']
    assert 1 <= rec['sweeps'] <= 4 and rec['objective'] < rec['objective_causal']
