"""Stage II with the Geman-McClure data term (``robust_data_sigma``; mosh2_options.robust_sigma): the reference's ``GMOf``
(scan2mesh/robustifiers.py:33-100) on every coordinate of every data row, psi(e) = sigma e / sqrt(sigma^2 + e^2), Jacobian rows
scaled by psi'(e) = (sigma^2 / (sigma^2 + e^2))^(3/2).

The float64 oracle is ``oracle.stageii`` with ``robust_data_sigma``; its closed form is ``oracle.robust``.

CPU: the closed form against golden vectors of the unmodified reference (tests/golden/ref_gmof.npz, written by
tests/golden/make_gmof_vectors.py), the oracle's Jacobian
against finite differences, the device source (single-thread host build) against the oracle on corrupted captures, the
recovery of a corrupted capture, and the plumbing of the keyword.  ``-m gpu``: the CUDA library against the oracle, the
default fast mode on a corrupted 500-frame capture, and the batch / subjects entry points against per-capture calls."""
import copy
import ctypes as C
import os

import numpy as np
import pytest

from conftest import dense_obs, run_oracle
from moshpp_b200 import build, chmosh, lib
from moshpp_b200.mocap_interface import MocapSession
from oracle import stageii as oracle_stageii
from oracle.robust import gm_dpsi, gm_psi

HERE = os.path.dirname(os.path.abspath(__file__))
SIGMA = 0.03        # metres: a few times the marker noise, well below a swapped label or a ghost marker


def run_robust_oracle(case, sigma, obs, vis, **kw):
    """The robust oracle on the dense observations ``obs`` / ``vis`` (latent-label order, metres)."""
    mocap = MocapSession(case['mocap_fname'], case['cfg'].mocap.unit)
    mocap.markers = np.where(vis[..., None], obs, 0.0)
    mocap.labels = list(case['latent_labels'])
    return run_oracle(case, mocap=mocap, robust_data_sigma=sigma, **kw)


# ---- corrupted captures -----------------------------------------------------------------------------------------------------
def corrupt(obs, vis, swap, ghost, spikes, seed=0):
    """A copy of a capture with two labels swapped over the frames ``swap``, one label replaced by a point 0.3 m away over the
    frames ``ghost`` and isolated 0.1 m spikes on single samples of the frames ``spikes``.  Returns (obs, vis, bad frames)."""
    rng = np.random.default_rng(seed)
    obs, vis = obs.copy(), vis.copy()
    F, M = vis.shape
    bad = np.zeros(F, dtype=bool)
    f0 = swap.start
    d = np.linalg.norm(obs[f0][:, None] - obs[f0][None], axis=-1)
    d[~vis[f0]] = 0
    d[:, ~vis[f0]] = 0
    far = min(0.25, 0.5 * d.max())                              # two labels >= 25 cm apart (on a hand: half its span)
    i, j = np.unravel_index(np.argmax(np.where(d > far, rng.random(d.shape), -1)), d.shape)
    obs[swap, i], obs[swap, j] = obs[swap, j].copy(), obs[swap, i].copy()
    vis[swap, i], vis[swap, j] = vis[swap, j].copy(), vis[swap, i].copy()
    bad[swap] = True
    k = (i + j + 1) % M if (i + j + 1) % M not in (i, j) else (i + j + 2) % M
    u = rng.normal(size=3)
    obs[ghost, k] += 0.3 * u / np.linalg.norm(u)
    bad[ghost] = True
    for f in spikes:
        m = int(rng.choice(np.flatnonzero(vis[f])))
        u = rng.normal(size=3)
        obs[f, m] += 0.1 * u / np.linalg.norm(u)
        bad[f] = True
    return obs, vis, bad


def small_corruption(case):
    """A short case's capture with a 3-frame swap, a 2-frame ghost marker and one spike."""
    obs, vis = dense_obs(case)
    F = len(obs)
    return corrupt(obs, vis, swap=slice(2, 5), ghost=slice(F - 3, F - 1), spikes=[F // 2 + 1])


# ---- the host build of the device source --------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def emu_handle():
    return C.CDLL(build.build_emu())


def case_options(case, sigma=0.0):
    pk, cfg = case['pack'], case['cfg']
    return lib.make_options(cfg.opt_settings.weights, optimize_fingers=bool(cfg.moshpp.optimize_fingers) and pk.finger_hi > pk.finger_lo,
                            optimize_dynamics=bool(cfg.moshpp.optimize_dynamics),
                            optimize_face=bool(cfg.moshpp.optimize_face) and pk.n_expr > 0, robust_sigma=sigma)


def emu_solve(handle, case, obs, vis, sigma, precision=lib.MOSH2_F64, chunk=(0, 0), entry='mosh2_emu_solve'):
    pk = case['pack']
    h = lib.DescHolder(pk)
    opt = case_options(case, sigma)
    res = lib.ResultArrays(len(obs), lib.pack_dims(pk))
    o = np.ascontiguousarray(obs, dtype=np.float64)
    v8 = np.ascontiguousarray(vis, dtype=np.uint8)
    sched = lib.make_schedule(*chunk)
    rc = getattr(handle, entry)(C.byref(h.desc), C.byref(opt), len(obs), o.ctypes.data_as(lib._f64p), v8.ctypes.data_as(lib._u8p),
                                C.byref(sched), precision, C.byref(res.c))
    assert rc == 0
    return res


def check_f64(case, res, out, tol_pose=1e-8, tol_trans=1e-9, rtol=1e-7):
    dbg = out['stageii_debug_details']
    fid = dbg['frame_ids']
    assert np.array_equal(np.nonzero(res.status & lib.ST_SOLVED)[0], fid)
    assert np.abs(res.pose[fid] - out['_pose_reduced']).max() < tol_pose
    assert np.abs(res.trans[fid] - out['trans']).max() < tol_trans
    if 'expression' in out:
        pk = case['pack']
        assert np.abs(res.dmpls[fid, pk.n_dmpl - pk.n_expr:pk.n_dmpl] - out['expression'][:, :pk.n_expr]).max() < tol_pose
    assert res.counters[fid, 2].sum() == dbg['oracle_stats']['j_evals']
    assert res.counters[fid, 3].sum() == dbg['oracle_stats']['minimizations']
    for col, k in enumerate(lib.ERR_NAMES):
        if k in dbg['stageii_errs'] and k not in ('velo', 'extrap_dmpl'):
            assert np.allclose(res.errs[fid, col], dbg['stageii_errs'][k], rtol=rtol, atol=1e-12), k


# ---- 1. golden pin -------------------------------------------------------------------------------------------------------------
def test_closed_form_equals_the_reference_gmof():
    """psi and psi' of the kernel's closed form against GMOf of the unmodified reference (GMOfInternal and SignedSqrt composed,
    values and compute_dr_wrt): relative 1e-12, and psi'(0) = 0 as the reference's SignedSqrt masks it."""
    z = np.load(os.path.join(HERE, 'golden', 'ref_gmof.npz'))
    for x, s, psi, dpsi in zip(z['x'], z['sigma'], z['psi'], z['dpsi']):
        assert np.allclose(gm_psi(x, s), psi, rtol=1e-12, atol=0)
        assert np.allclose(gm_dpsi(x, s), dpsi, rtol=1e-12, atol=0)
        assert (x == 0).sum() == 1 and (np.abs(x) == 1e-9).sum() == 2 and np.abs(x).max() >= 40 * s
        assert (dpsi[x == 0] == 0).all() and (gm_dpsi(x, s)[x == 0] == 0).all()
        assert dpsi[np.abs(x) == 1e-9].min() > 0.999 and np.abs(psi[np.abs(x) >= 10 * s]).min() > 0.99 * s


# ---- 2. oracle Jacobian --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', ['C2', 'CF'])
def test_oracle_robust_jacobian_matches_finite_differences(cases, name):
    case = cases(name)
    obs, vis, _ = small_corruption(case)
    solver = oracle_stageii.StageIISolver(case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'],
                                          robust_data_sigma=SIGMA)
    f = 3                                                        # a frame of the swap
    vi = np.flatnonzero(vis[f])
    rng = np.random.default_rng(1)
    solver.pose[:] = rng.normal(0, 0.1, solver.pose.shape)
    solver.trans[:] = obs[f, vi].mean(0)
    terms, _ = solver.frame_terms(len(vi), velo_target=np.zeros_like(solver.pose))
    obj = oracle_stageii._Objective(solver, obs[f, vi], vi, terms, solver.step2_ids, solver.nd > 0)
    x0 = obj.x0()
    r0, J = obj(x0, True)
    e = (solver.evaluate(False)['markers'][vi] - obs[f, vi]).reshape(-1)
    assert np.abs(e).max() > 5 * SIGMA and np.abs(e).min() < SIGMA      # saturated and unsaturated rows
    h = 1e-6
    Jfd = np.zeros_like(J)
    for c in range(len(x0)):
        xp, xm = x0.copy(), x0.copy()
        xp[c] += h
        xm[c] -= h
        Jfd[:, c] = (obj(xp, False) - obj(xm, False)) / (2 * h)
    assert np.abs(J - Jfd).max() / np.abs(J).max() < 5e-8


# ---- 3. the host build against the oracle ---------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', ['C1', 'C2', 'CF', 'C4'])
def test_f64_device_source_equals_robust_oracle(cases, emu_handle, name):
    """Bodies at sigma = 3 cm; the MANO hand (C4), whose markers lie 1-3 cm apart, at sigma = 1 cm.  (At 3 cm the hand's
    frame problem -- no pose prior, weakly observed finger coefficients -- leaves the host build and the oracle 2.3e-6 rad apart
    with identical iteration counts: rounding carried along nearly flat directions, not a difference of the objective.)"""
    case = cases(name)
    sigma = 0.01 if name == 'C4' else SIGMA
    obs, vis, _ = small_corruption(case)
    out = run_robust_oracle(case, sigma, obs, vis)
    res = emu_solve(emu_handle, case, obs, vis, sigma)
    check_f64(case, res, out)
    plain = emu_solve(emu_handle, case, obs, vis, 0.0)                  # the robust term does change the solve
    assert np.abs(plain.pose - res.pose).max() > 1e-3


def test_f32_device_source_within_tolerance(cases, emu_handle):
    case = cases('C2')
    obs, vis, _ = small_corruption(case)
    out = run_robust_oracle(case, SIGMA, obs, vis)
    res = emu_solve(emu_handle, case, obs, vis, SIGMA, precision=lib.MOSH2_F32)
    fid = out['stageii_debug_details']['frame_ids']
    bd = case['pack'].body_dof
    dp = np.abs(res.pose[fid] - out['_pose_reduced'])
    assert dp[:, :bd].max() < 1e-3 and dp.max() < 5e-3
    assert np.abs(res.trans[fid] - out['trans']).max() < 1e-4
    sse = out['stageii_debug_details']['stageii_errs']['data']
    assert np.abs(res.errs[fid, 0] / sse - 1).max() < 1e-2


def test_chunked_schedule_matches_robust_oracle_chunked(cases, emu_handle):
    case = cases('C2')
    obs, vis, _ = small_corruption(case)
    out = run_robust_oracle(case, SIGMA, obs, vis, chunk=(5, 2))
    res = emu_solve(emu_handle, case, obs, vis, SIGMA, chunk=(5, 2))
    fid = out['stageii_debug_details']['frame_ids']
    assert np.abs(res.pose[fid] - out['_pose_reduced']).max() < 1e-8
    assert np.abs(res.trans[fid] - out['trans']).max() < 1e-9


def test_resumed_chunks_equal_robust_oracle_sequential(cases, emu_handle):
    """Cold-started chunks without warm-up, then every chunk resumed in order (boundary repair): the robust sequential pass."""
    case = cases('C2')
    obs, vis, _ = small_corruption(case)
    out = run_robust_oracle(case, SIGMA, obs, vis)
    seq = emu_solve(emu_handle, case, obs, vis, SIGMA)
    res = emu_solve(emu_handle, case, obs, vis, SIGMA, chunk=(3, 0, -1), entry='mosh2_emu_solve_resumed')
    assert np.array_equal(res.pose, seq.pose) and np.array_equal(res.errs, seq.errs)
    check_f64(case, res, out)


# ---- 4. corrupted-capture recovery ----------------------------------------------------------------------------------------------
def test_robust_solve_recovers_a_corrupted_capture(cases, emu_handle):
    """A 160-frame C2 capture with a 40-frame label swap, a 30-frame ghost marker and six isolated 0.1 m spikes, solved in
    float64 on the host build with the least-squares and the robust data term.  The error of a solve is measured against the
    least-squares solve of the clean capture: the synthetic model's ground-truth pose is itself only recovered to ~0.6 rad on
    its worst body coefficient from 53 markers, which would mask the effect of the corruption.  Measured on the first run:
    worst body-pose error on the corrupted frames 2.15 rad (L2) against 0.49 rad (robust), a ratio of 0.23; on the clean frames
    (16 frames or more behind every corruption) the two solves agree to 2.6e-3 rad.  The bounds below (1/4, 5e-3 rad) are set
    from that run."""
    case = cases('C2', frames=160)
    obs0, vis0 = dense_obs(case)
    obs, vis, bad = corrupt(obs0, vis0, swap=slice(20, 60), ghost=slice(80, 110), spikes=[10, 65, 70, 120, 135, 150])
    ref = emu_solve(emu_handle, case, obs0, vis0, 0.0)
    l2 = emu_solve(emu_handle, case, obs, vis, 0.0)
    rb = emu_solve(emu_handle, case, obs, vis, SIGMA)
    bd = case['pack'].body_dof
    e_l2 = np.abs(l2.pose[:, :bd] - ref.pose[:, :bd]).max(1)
    e_rb = np.abs(rb.pose[:, :bd] - ref.pose[:, :bd]).max(1)
    # clean frames: those the corruption does not reach through the velocity term either (a few frames after each event)
    near = np.convolve(bad.astype(float), np.ones(16), mode='full')[:len(bad)] > 0
    clean = ~near
    print(f'\nworst body error on corrupted frames: L2 {e_l2[bad].max():.4g} rad, robust {e_rb[bad].max():.4g} rad; '
          f'clean frames robust vs L2 {np.abs(rb.pose[clean, :bd] - l2.pose[clean, :bd]).max():.3g} rad')
    assert e_rb[bad].max() <= 0.25 * e_l2[bad].max()
    assert np.abs(rb.pose[clean, :bd] - l2.pose[clean, :bd]).max() < 5e-3


# ---- 5. plumbing -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('sigma', [0.0, -0.01, float('nan'), float('inf')])
def test_entry_points_reject_a_bad_sigma(cases, sigma):
    case = cases('C1')
    args = (case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])
    with pytest.raises(ValueError, match='robust_data_sigma'):
        chmosh.mosh_stageii(case['mocap_fname'], *args, robust_data_sigma=sigma)
    with pytest.raises(ValueError, match='robust_data_sigma'):
        chmosh.mosh_stageii_batch([case['mocap_fname']], *args, robust_data_sigma=sigma)
    subject = dict(cfg=case['cfg'], mocap_fnames=[case['mocap_fname']], markers_latent=case['markers_latent'],
                   latent_labels=case['latent_labels'], betas=case['betas'], marker_meta=case['marker_meta'])
    with pytest.raises(ValueError, match='robust_data_sigma'):
        chmosh.mosh_stageii_subjects([subject], robust_data_sigma=sigma)
    with pytest.raises(ValueError, match='robust_data_sigma'):
        chmosh.mosh_stageii_subjects([dict(subject, robust_data_sigma=sigma)])


def test_sigma_reaches_the_options_and_leaves_the_cached_ones(cases):
    case = cases('C1')
    cap = dict(F=case['pack'].n_markers)
    sub = chmosh._subject([cap], case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'], None,
                          0, subject_cache=False, robust_data_sigma=0.025)
    assert sub['opts'].robust_sigma == 0.025 and sub['robust_data_sigma'] == 0.025
    _, opts, _ = chmosh.prepare_stageii(case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])
    o = chmosh.with_robust_sigma(opts, 0.025)
    assert o is not opts and o.robust_sigma == 0.025 and opts.robust_sigma == 0.0
    assert chmosh.with_robust_sigma(opts, None) is opts
    for f, _ in lib.Options._fields_:
        if f != 'robust_sigma':
            assert getattr(o, f) == getattr(opts, f), f


def test_subjects_with_other_sigma_get_their_own_launch(cases):
    case = cases('C2')
    pk, opts, _ = chmosh.prepare_stageii(case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])
    keys = [chmosh.subject_launch_key(pk, chmosh.with_robust_sigma(opts, s)) for s in (None, 0.03, 0.03, 0.05, None)]
    assert chmosh.launch_groups(keys) == [[0, 4], [1, 2], [3]]


def test_library_default_options_turn_the_robust_term_off():
    o = lib.Options()
    o.robust_sigma = 1.0
    lib.load_library().mosh2_default_options(C.byref(o))
    assert o.robust_sigma == 0.0


def test_options_without_sigma_are_byte_identical_to_the_previous_abi(cases):
    """mosh2_options of ABI 107 (without robust_sigma) and of this ABI with sigma None: the same bytes, then a zero double."""
    class Options107(C.Structure):
        _fields_ = [f for f in lib.Options._fields_ if f[0] != 'robust_sigma']
    assert lib.Options._fields_[-1] == ('robust_sigma', C.c_double)
    case = cases('CF')
    _, opts, _ = chmosh.prepare_stageii(case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])
    opts = chmosh.with_robust_sigma(opts, None)
    old = Options107(**{f: getattr(opts, f) for f, _ in Options107._fields_})
    new = bytes(opts)
    assert C.sizeof(lib.Options) == C.sizeof(Options107) + 8 and C.sizeof(Options107) % 8 == 0
    assert new[:C.sizeof(Options107)] == bytes(old) and new[C.sizeof(Options107):] == bytes(8)
    assert bytes(lib.make_options()) == bytes(lib.make_options(robust_sigma=0.0))


# ---- GPU ---------------------------------------------------------------------------------------------------------------------------
def _args(case):
    return (case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])


def write_capture(case, obs, vis, fname):
    """The capture ``obs`` / ``vis`` (latent-label order, metres) as an npz mocap file in millimetres (missing = NaN)."""
    np.savez(fname, markers=np.where(vis[..., None], obs, np.nan) * 1000.0, labels=np.array(case['latent_labels']), frame_rate=120.0)
    cfg = copy.deepcopy(case['cfg'])
    cfg.mocap.fname = fname
    return cfg


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['C2', 'CF'])
def test_f64_kernel_equals_robust_oracle(cases, name):
    case = cases(name)
    obs, vis, _ = small_corruption(case)
    out = run_robust_oracle(case, SIGMA, obs, vis)
    pk, opts, _ = chmosh.prepare_stageii(*_args(case))
    model = lib.Model(pk, device=0)
    try:
        res = model.solve(obs, vis, chmosh.with_robust_sigma(opts, SIGMA), chunk_len=0, precision=lib.MOSH2_F64)
    finally:
        model.close()
    check_f64(case, res, out)


@pytest.mark.gpu
def test_default_fast_mode_on_a_corrupted_capture(cases, tmp_path):
    """The default path (float32, planned chunks, verified warm-up) with the robust term on a corrupted 500-frame C2 capture,
    against the robust sequential float64 solve of the same library (which test_f64_kernel_equals_robust_oracle ties to the
    oracle): BASELINE.md section 4's fast-mode tolerances."""
    case = cases('C2', frames=500)
    obs0, vis0 = dense_obs(case)
    obs, vis, bad = corrupt(obs0, vis0, swap=slice(100, 140), ghost=slice(300, 330), spikes=[30, 200, 250, 420, 470])
    fn = str(tmp_path / 'corrupted_C2.npz')
    cfg = write_capture(case, obs, vis, fn)
    args = (cfg,) + _args(case)[1:]
    fast = chmosh.mosh_stageii(fn, *args, robust_data_sigma=SIGMA)
    ref = chmosh.mosh_stageii(fn, *args, robust_data_sigma=SIGMA, precision='f64', chunk_len=0)
    b, rb = fast['stageii_debug_details']['b200'], ref['stageii_debug_details']['b200']
    assert b['precision'] == 'f32' and b['chunks'] > 1 and b['robust_data_sigma'] == SIGMA
    assert np.array_equal(b['frame_ids'], rb['frame_ids'])
    bd = min(case['pack'].body_dof, 66)
    dp = np.abs(b['pose_reduced'] - rb['pose_reduced'])
    body, dtr = dp[:, :bd].max(1), np.abs(fast['trans'] - ref['trans']).max(1)
    sse = fast['stageii_debug_details']['stageii_errs']['data'] / ref['stageii_debug_details']['stageii_errs']['data']
    print(f'\nfast vs f64 sequential: body over 1e-3 rad on {(body > 1e-3).sum()} frames (max {body.max():.3g}), trans over 1e-4 m '
          f'on {(dtr > 1e-4).sum()}, data SSE outside 1 % on {(np.abs(sse - 1) > 1e-2).sum()}')
    assert (body > 1e-3).mean() <= 0.01 and (dtr > 1e-4).mean() <= 0.01 and (np.abs(sse - 1) > 1e-2).mean() <= 0.01
    assert body.max() < 0.05 and dtr.max() < 2e-3


@pytest.mark.gpu
def test_batch_and_subjects_equal_per_capture_calls(tmp_path):
    from moshpp_b200 import synth
    case, fnames = synth.make_subject(str(tmp_path / 'subject'), 'C2', (40, 24), n_verts=1500)
    kw = dict(precision='f64', chunk_len=0, robust_data_sigma=SIGMA)
    one = [chmosh.mosh_stageii(fn, *_args(case), **kw) for fn in fnames]
    plain = chmosh.mosh_stageii(fnames[0], *_args(case), precision='f64', chunk_len=0)
    assert np.abs(plain['fullpose'] - one[0]['fullpose']).max() > 0
    batch = chmosh.mosh_stageii_batch(fnames, *_args(case), **kw)
    subject = dict(cfg=case['cfg'], mocap_fnames=fnames, markers_latent=case['markers_latent'], latent_labels=case['latent_labels'],
                   betas=case['betas'], marker_meta=case['marker_meta'])
    subs = chmosh.mosh_stageii_subjects([subject, dict(subject, robust_data_sigma=None)], **kw)
    assert subs[0][0]['stageii_debug_details']['b200']['batch']['launches'] == 2
    for got in (batch, subs[0]):
        for a, b in zip(got, one):
            assert np.array_equal(a['fullpose'], b['fullpose']) and np.array_equal(a['trans'], b['trans'])
            for k, v in b['stageii_debug_details']['stageii_errs'].items():
                assert np.array_equal(a['stageii_debug_details']['stageii_errs'][k], v), k
            assert a['stageii_debug_details']['b200']['robust_data_sigma'] == SIGMA
    assert np.array_equal(subs[1][0]['fullpose'], plain['fullpose'])
    assert 'robust_data_sigma' not in subs[1][0]['stageii_debug_details']['b200']       # (the b200 keys of a call without it)
