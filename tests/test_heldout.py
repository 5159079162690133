"""Held-out marker validation of Stage II (``mosh_stageii(..., heldout=...)``; DESIGN.md section 12).

A fold's solve is Stage II on the capture with every sample of the fold's markers deleted; the error of a held-out marker is
the distance of its simulated position on the fold's solved body from where the camera saw it.  The fold gather and the
held-out error of the device source run here through its host build (tests/emu/mosh2_emu_heldout.cpp) and are checked against
host masking and the float64 oracle (``oracle.heldout``); the GPU tests run the CUDA kernels through ``mosh_stageii``.
"""
from __future__ import annotations

import copy
import ctypes as C
import os
import time

import numpy as np
import pytest

from moshpp_b200 import build, chmosh, lib
from moshpp_b200.mocap_interface import MocapSession, load_markers, rotation_xyz
from oracle import heldout as oracle_heldout

E_INVALID = -1          # MOSH2_E_INVALID


@pytest.fixture(scope='module')
def emu_lib():
    h = C.CDLL(build.build_emu())
    h.mosh2_emu_upload_markers_folds.argtypes = [C.c_int32, C.c_int32, C.c_int32, lib._i32p, lib._f64p, lib._u8p, lib._f64p, lib._i32p,
                                                 C.c_int32, C.c_int32, lib._f64p, C.c_int32, C.c_int32, lib._i32p, lib._u8p, C.c_int32,
                                                 C.c_int32, C.c_double, lib._f64p]
    h.mosh2_emu_heldout_errors.argtypes = [C.c_int32, C.c_int32, C.c_int32, lib._u8p, C.c_int32, lib._f64p, lib._i32p, lib._f64p,
                                           lib._f64p, lib._i32p]
    h.mosh2_emu_upload_markers_range.argtypes = [C.c_int32, C.c_int32, C.c_int32, lib._f64p, lib._u8p, C.c_int32, C.c_int32, lib._f64p,
                                                 C.c_int32, C.c_int32, lib._i32p, C.c_int32, C.c_int32, C.c_double, lib._f64p]
    return h


def emu_folds(h, precision, M, counts, seq0, hide, raw, cols, start, step, unit, rot):
    """mosh2_emu_upload_markers_folds -> (rc, obs, vis, side)."""
    counts = np.ascontiguousarray(counts, dtype=np.int32)
    F, n = int(counts.sum()), int(counts[seq0]) if 0 <= seq0 < len(counts) else 1
    hide8 = np.ascontiguousarray(hide, dtype=np.uint8)
    K = max(int(hide8.sum(1).max()), 1)
    obs, vis = np.full((F, M, 3), np.nan), np.full((F, M), 7, dtype=np.uint8)
    side = np.full((hide8.shape[0], n, K, 3), -1.0)
    k_out = C.c_int32()
    raw = np.ascontiguousarray(raw, dtype=np.float64)
    cols = np.ascontiguousarray(cols, dtype=np.int32)
    r = None if rot is None else np.ascontiguousarray(rot, dtype=np.float64)
    rc = h.mosh2_emu_upload_markers_folds(precision, M, len(counts), lib._ptr(counts, lib._i32p), lib._ptr(obs, lib._f64p),
                                          lib._ptr(vis, lib._u8p), lib._ptr(side, lib._f64p), C.byref(k_out), seq0, hide8.shape[0],
                                          lib._ptr(raw, lib._f64p), raw.shape[0], raw.shape[1], lib._ptr(cols, lib._i32p),
                                          lib._ptr(hide8, lib._u8p), start, step, unit, lib._ptr(r, lib._f64p) if r is not None else None)
    return rc, obs, vis, side


def emu_range(h, precision, M, n, raw, cols, start, step, unit, rot):
    """The capture through mosh2_emu_upload_markers_range (the device adapter's rule) -> (obs, vis) of n frames."""
    obs, vis = np.zeros((n, M, 3)), np.zeros((n, M), dtype=np.uint8)
    raw = np.ascontiguousarray(raw, dtype=np.float64)
    cols = np.ascontiguousarray(cols, dtype=np.int32)
    r = None if rot is None else np.ascontiguousarray(rot, dtype=np.float64)
    assert h.mosh2_emu_upload_markers_range(precision, M, n, lib._ptr(obs, lib._f64p), lib._ptr(vis, lib._u8p), 0, n, lib._ptr(raw, lib._f64p),
                                            raw.shape[0], raw.shape[1], lib._ptr(cols, lib._i32p), start, step, unit,
                                            lib._ptr(r, lib._f64p) if r is not None else None) == 0
    return obs, vis.astype(bool)


def masked(obs, vis, hide):
    """Host masking of a capture's observations: per fold obs / vis with the hidden markers missing, and the side buffer."""
    K = int(hide.sum(1).max())
    fo = np.repeat(obs[None], len(hide), 0)
    fv = np.repeat(vis[None], len(hide), 0)
    side = np.full((len(hide), len(obs), K, 3), np.nan)
    for k, h in enumerate(hide):
        idx = np.flatnonzero(h)
        fo[k][:, idx] = 0.0
        fv[k][:, idx] = False
        side[k, :, :len(idx)] = np.where(vis[:, idx, None], obs[:, idx], np.nan)
    return fo.reshape(-1, *obs.shape[1:]), fv.reshape(-1, vis.shape[1]), side


# ---- fold gather ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('precision', [lib.MOSH2_F64, lib.MOSH2_F32])
@pytest.mark.parametrize('variant', ['mm', 'rotate', 'absent_label'])
def test_fold_gather_equals_host_masking(cases, tmp_path, emu_lib, precision, variant):
    case = cases('C1')           # (c3d, millimetres, NaN gaps, an extra label)
    labels = list(case['latent_labels'])
    M = len(labels)
    fn, rot = case['mocap_fname'], None
    if variant == 'rotate':
        rot = [10.0, -20.0, 30.0]
    if variant == 'absent_label':                # a latent label the file does not have
        raw0, raw_labels, _ = load_markers(fn)
        keep = [c for c, l in enumerate(raw_labels) if l != labels[3]]
        fn = str(tmp_path / 'absent.npz')
        np.savez(fn, markers=raw0[:, keep], labels=np.array(raw_labels)[keep], frame_rate=120.0)
    m = MocapSession(fn, case['cfg'].mocap.unit, mocap_rotate=rot)
    cols = m.raw_columns_for_labels(labels)
    assert (variant == 'absent_label') == (cols[3] < 0)
    sel = range(1, len(m), 2)
    R = None if rot is None else rotation_xyz(rot)
    hide = np.zeros((3, M), dtype=bool)
    hide[0, 3] = True
    hide[1, [0, 5, 7]] = True
    hide[2, [M - 1]] = True
    counts = [4] + [len(sel)] * 3                # the folds behind another sequence of the job
    rc, obs, vis, side = emu_folds(emu_lib, precision, M, counts, 1, hide, m.raw, cols, sel.start, sel.step, m.unit_per_metre, R)
    assert rc == 0
    o, v = emu_range(emu_lib, lib.MOSH2_F64, M, len(sel), m.raw, cols, sel.start, sel.step, m.unit_per_metre, R)
    want_obs, want_vis, want_side = masked(o, v, hide)
    if precision == lib.MOSH2_F32:
        want_obs = want_obs.astype(np.float32).astype(np.float64)
    assert np.array_equal(vis[4:].astype(bool), want_vis) and set(np.unique(vis[4:])) == {0, 1}
    assert np.array_equal(obs[4:], want_obs)
    for k, h in enumerate(hide):                                     # (float64 whatever the job's precision)
        assert np.array_equal(side[k, :, :h.sum()], want_side[k, :, :h.sum()], equal_nan=True)
    assert np.isnan(obs[:4]).all() and (vis[:4] == 7).all()          # the other sequence is not touched
    # and the host adapter of the product, up to the rounding of the rotation
    ho, hv = m.frames_for_labels(labels, sel)
    assert np.array_equal(v, hv) and np.abs(o - ho).max() < 1e-12
    if variant == 'absent_label':
        assert np.isnan(side[0, :, 0]).all()


def test_fold_upload_checks(emu_lib):
    raw = np.ones((10, 4, 3))
    cols, M = [0, 3], 2
    hide = np.array([[1, 0], [0, 1]])
    ok = lambda counts, seq0, hide, start=0, step=1: emu_folds(emu_lib, 1, M, counts, seq0, hide, raw, cols, start, step, 1.0, None)[0]
    assert ok([6, 6], 0, hide) == 0
    assert ok([3, 6, 6], 1, hide) == 0
    assert ok([6, 5], 0, hide) == E_INVALID                          # folds of different frame counts: a job of the wrong shape
    assert ok([6, 6], 1, hide) == E_INVALID                          # past the job's sequences
    assert ok([6, 6], 0, np.array([[1, 0], [0, 0]])) == E_INVALID    # a fold that hides nothing
    assert ok([6, 6], 0, np.array([[1, 0], [0, 2]])) == E_INVALID    # a mask that is not 0 / 1
    assert ok([6, 6], 0, hide, start=5) == E_INVALID                 # past the file's frames


# ---- fold solve and errors against the oracle -------------------------------------------------------------------------------
def capture_with(case, tmp_path, name, edit):
    """The case's capture file rewritten as it is (file units, missing = NaN) after ``edit(markers [F, L, 3], labels)``; returns
    (file name, cfg)."""
    raw, labels, _ = load_markers(case['mocap_fname'])
    mk = np.array(raw, dtype=np.float64)
    edit(mk, list(labels))
    fn = str(tmp_path / f'{name}.npz')
    np.savez(fn, markers=mk, labels=np.array(labels), frame_rate=120.0)
    cfg = copy.deepcopy(case['cfg'])
    cfg.mocap.fname = fn
    return fn, cfg


def case_options(case, robust_sigma=0.0):
    pk, cfg = case['pack'], case['cfg']
    return lib.make_options(cfg.opt_settings.weights, optimize_fingers=bool(cfg.moshpp.optimize_fingers) and pk.finger_hi > pk.finger_lo,
                            optimize_dynamics=bool(cfg.moshpp.optimize_dynamics),
                            optimize_face=bool(cfg.moshpp.optimize_face) and pk.n_expr > 0, robust_sigma=robust_sigma)


def emu_heldout(h, case, fn, cfg, hide, robust_sigma=0.0):
    """The folds of the capture ``fn`` through the host build: fold gather, one sequential batch solve in float64, held-out
    errors.  Returns (err [n_folds, F, K], fold status [n_folds, F], Jacobian builds per fold)."""
    labels = list(case['latent_labels'])
    M, n_folds = len(labels), len(hide)
    m = MocapSession(fn, cfg.mocap.unit, mocap_rotate=cfg.mocap.rotate)
    F = len(m)
    rc, obs, vis, side = emu_folds(h, lib.MOSH2_F64, M, [F] * n_folds, 0, hide, m.raw, m.raw_columns_for_labels(labels), 0, 1,
                                   m.unit_per_metre, None)
    assert rc == 0
    pk = case['pack']
    d = lib.DescHolder(pk)
    opt = case_options(case, robust_sigma)
    counts = np.full(n_folds, F, dtype=np.int32)
    res = lib.ResultArrays(F * n_folds, lib.pack_dims(pk))
    sched = lib.make_schedule(0, 0)
    v8 = np.ascontiguousarray(vis, dtype=np.uint8)
    assert h.mosh2_emu_solve_batch(C.byref(d.desc), C.byref(opt), n_folds, lib._ptr(counts, lib._i32p), lib._ptr(obs, lib._f64p),
                                   lib._ptr(v8, lib._u8p), C.byref(sched), lib.MOSH2_F64, C.byref(res.c)) == 0
    K = int(hide.sum(1).max())
    err, st = np.zeros((n_folds, F, K)), np.zeros((n_folds, F), dtype=np.int32)
    hide8 = np.ascontiguousarray(hide, dtype=np.uint8)
    sim = np.ascontiguousarray(res.markers_sim)
    assert h.mosh2_emu_heldout_errors(M, n_folds, F, lib._ptr(hide8, lib._u8p), 0, lib._ptr(sim, lib._f64p), lib._ptr(res.status, lib._i32p),
                                      lib._ptr(side, lib._f64p), lib._ptr(err, lib._f64p), lib._ptr(st, lib._i32p)) == 0
    builds = res.counters[:, 2].reshape(n_folds, F).sum(1)
    return err, st, builds


def oracle_folds(case, fn, cfg, hide, robust_sigma=None):
    labels = list(case['latent_labels'])
    return oracle_heldout.heldout_errors(fn, cfg, case['markers_latent'], labels, case['betas'], case['marker_meta'],
                                         [[labels[i] for i in np.flatnonzero(h)] for h in hide], robust_data_sigma=robust_sigma)


def dropout(col_of, lo, hi):
    def edit(mk, labels):
        mk[lo:hi, col_of(labels)] = np.nan
    return edit


@pytest.mark.parametrize('name,sigma', [('C1', None), ('C2', None), ('CF', None), ('C2', 0.03)])
def test_fold_errors_match_oracle(cases, tmp_path, emu_lib, name, sigma):
    case = cases(name)
    labels = list(case['latent_labels'])
    M = len(labels)
    edit = dropout(lambda L: [L.index(labels[2]), L.index(labels[9])], 5, 9) if name == 'C2' else (lambda mk, L: None)
    fn, cfg = capture_with(case, tmp_path, f'{name}_{sigma}', edit)
    hide = np.zeros((3, M), dtype=bool)
    hide[0, 2] = True                         # (C2: a marker with a dropout of its own)
    hide[1, [4, M - 1]] = True                # two markers of one fold
    hide[2, M // 2] = True
    err, st, builds = emu_heldout(emu_lib, case, fn, cfg, hide, sigma or 0.0)
    ref = oracle_folds(case, fn, cfg, hide, sigma)
    assert np.array_equal(np.isnan(err), np.isnan(ref['err']))
    assert np.nanmax(np.abs(err - ref['err'])) < 1e-9
    assert np.array_equal(builds, ref['j_evals'])
    for k in range(len(hide)):
        assert np.array_equal(np.flatnonzero(st[k] & lib.ST_SOLVED), ref['frame_ids'][k])
    if name == 'C2':                          # the dropout of the held-out marker: no error there
        assert np.isnan(err[0, 5:9, 0]).all() and np.isfinite(err[0, 9:, 0]).sum() >= 5


def only_one_visible(case, tmp_path, keep, frame=3):
    """The case's capture with every marker but ``keep`` missing in ``frame``."""
    labels = list(case['latent_labels'])

    def edit(mk, L):
        cols = [c for c, l in enumerate(L) if l != labels[keep]]
        mk[frame, cols] = np.nan
    return capture_with(case, tmp_path, 'only_one', edit)


def test_fold_of_only_visible_marker_skips_the_frame(cases, tmp_path, emu_lib):
    case = cases('C1')
    M = len(case['latent_labels'])
    _, vis = MocapSession(case['mocap_fname'], case['cfg'].mocap.unit).frames_for_labels(case['latent_labels'], range(4))
    keep, other = np.flatnonzero(vis[3])[:2]
    fn, cfg = only_one_visible(case, tmp_path, keep=keep)
    hide = np.zeros((2, M), dtype=bool)
    hide[0, keep] = True
    hide[1, other] = True
    err, st, _ = emu_heldout(emu_lib, case, fn, cfg, hide)
    ref = oracle_folds(case, fn, cfg, hide)
    assert not (st[0, 3] & lib.ST_SOLVED) and (st[0, 3] & lib.ST_SKIPPED) and np.isnan(err[0, 3]).all()
    assert 3 not in ref['frame_ids'][0] and np.isnan(ref['err'][0, 3]).all()
    assert (st[1, 3] & lib.ST_SOLVED) and np.isnan(err[1, 3, 0])       # the other fold solves it; `other` is not observed there
    assert np.isfinite(err[0, :3, 0]).all()


# ---- keyword -----------------------------------------------------------------------------------------------------------------
def test_heldout_keyword(cases):
    case = cases('C1')
    labels = list(case['latent_labels'])
    assert chmosh.check_heldout(None, labels) is None
    assert chmosh.check_heldout('each', labels) == 'each'
    assert chmosh.check_heldout([[labels[3], labels[1]], (labels[2],)], labels) == [[1, 3], [2]]
    args = (case['mocap_fname'], case['cfg'], case['markers_latent'], labels, case['betas'], case['marker_meta'])
    for bad in ('all', 'EACH', [], [[]], [labels[0]], [['no_such_label']], [[labels[0]], ['no_such_label']], 3, True, {'a': 1},
                [[labels[0], 7]]):
        with pytest.raises(ValueError):
            chmosh.mosh_stageii(*args, heldout=bad)          # (raised before any capture is read or any device is asked for)


# ---- GPU ------------------------------------------------------------------------------------------------------------------------
def _outputs_equal(a, b):
    """The output dictionaries of two Stage-II calls, byte for byte, apart from b200 (timings)."""
    assert set(a) == set(b)
    for k in a:
        if k == 'stageii_debug_details':
            da, db = a[k], b[k]
            assert set(da) == set(db)
            for q in da:
                if q == 'b200':
                    for f in ('status', 'counters', 'pose_reduced', 'frame_ids'):
                        assert np.asarray(da[q][f]).tobytes() == np.asarray(db[q][f]).tobytes(), f
                elif q in ('markers_sim', 'markers_obs'):
                    assert len(da[q]) == len(db[q]) and all(x.tobytes() == y.tobytes() for x, y in zip(da[q], db[q]))
                elif q == 'stageii_errs':
                    assert set(da[q]) == set(db[q]) and all(da[q][e].tobytes() == db[q][e].tobytes() for e in da[q])
                elif isinstance(da[q], np.ndarray):
                    assert da[q].tobytes() == db[q].tobytes()
                else:
                    assert da[q] == db[q], q
        else:
            assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes(), k


@pytest.mark.gpu
def test_gpu_main_result_unchanged(cases):
    case = cases('C2')
    args = (case['mocap_fname'], case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])
    off = chmosh.mosh_stageii(*args)
    on = chmosh.mosh_stageii(*args, heldout='each')
    _outputs_equal(off, on)
    assert 'heldout' not in off['stageii_debug_details']['b200']
    h = on['stageii_debug_details']['b200']['heldout']
    assert h['device_errors'] and len(h['folds']) == len(case['latent_labels'])
    assert h['err'].shape == (len(h['labels']), len(off['fullpose']))
    assert h['overall']['n'] > 0 and np.isfinite(h['overall']['mean']) and h['visible']['overall']['n'] > 0


@pytest.mark.gpu
def test_gpu_float64_errors_match_oracle(cases, tmp_path):
    case = cases('C2')
    labels = list(case['latent_labels'])
    M = len(labels)
    fn, cfg = capture_with(case, tmp_path, 'c2_dropout', dropout(lambda L: [L.index(labels[2]), L.index(labels[9])], 5, 9))
    folds = [[labels[2]], [labels[4], labels[M - 1]], [labels[M // 2]]]
    out = chmosh.mosh_stageii(fn, cfg, case['markers_latent'], labels, case['betas'], case['marker_meta'], chunk_len=0, precision='f64',
                              heldout=folds)
    h = out['stageii_debug_details']['b200']['heldout']
    hide = np.zeros((3, M), dtype=bool)
    for k, f in enumerate(folds):
        hide[k, [labels.index(l) for l in f]] = True
    ref = oracle_folds(case, fn, cfg, hide)
    fid = out['stageii_debug_details']['b200']['frame_ids']
    want = np.concatenate([ref['err'][k][fid][:, :hide[k].sum()].T for k in range(3)])
    assert h['labels'] == [labels[2], labels[4], labels[M - 1], labels[M // 2]]
    assert np.array_equal(np.isnan(h['err']), np.isnan(want)) and np.nanmax(np.abs(h['err'] - want)) < 1e-8
    # and through the host adapter (a frame selection that is not a forward range inside the file is not one; device_adapter off)
    out2 = chmosh.mosh_stageii(fn, cfg, case['markers_latent'], labels, case['betas'], case['marker_meta'], chunk_len=0, precision='f64',
                               heldout=folds, device_adapter=False)
    h2 = out2['stageii_debug_details']['b200']['heldout']
    assert not h2['device_errors'] and np.nanmax(np.abs(h2['err'] - want)) < 1e-8


@pytest.mark.gpu
def test_gpu_skipped_frame_and_fold(cases, tmp_path):
    case = cases('C1')
    labels = list(case['latent_labels'])
    _, vis = MocapSession(case['mocap_fname'], case['cfg'].mocap.unit).frames_for_labels(labels, range(4))
    keep = int(np.flatnonzero(vis[3])[0])

    def capture(never):
        def edit(mk, L):
            mk[3, [c for c, l in enumerate(L) if l != labels[keep]]] = np.nan   # frame 3: one marker alone
            mk[:, [c for c, l in enumerate(L) if l == labels[never]]] = np.nan  # a label the capture never observes
        fn, cfg = capture_with(case, tmp_path, f'never{never}', edit)
        m = MocapSession(fn, cfg.mocap.unit, labels_map='general')               # (the label clean-up of mosh_stageii)
        return fn, cfg, not m.frames_for_labels(labels, range(len(m)))[1][:, never].any()

    # a label whose only source is its own column (another raw label may be a synonym of it)
    never, (fn, cfg, ok) = next((q, r) for q in range(len(labels)) if q != keep for r in [capture(q)] if r[2])
    assert ok
    out = chmosh.mosh_stageii(fn, cfg, case['markers_latent'], labels, case['betas'], case['marker_meta'], heldout='each')
    h = out['stageii_debug_details']['b200']['heldout']
    assert [labels[never]] not in h['folds'] and [labels[never]] in h['skipped_folds']
    k = h['folds'].index([labels[keep]])
    assert h['fold_status'][k]['skipped'] == 1 and all(s['skipped'] == 0 for q, s in enumerate(h['fold_status']) if q != k)
    fid = list(out['stageii_debug_details']['b200']['frame_ids'])
    assert np.isnan(h['err'][h['labels'].index(labels[keep]), fid.index(3)])


@pytest.mark.gpu
@pytest.mark.parametrize('sweeps', [None, 4])
def test_gpu_fold_rows_equal_batch_of_missing_files(cases, tmp_path, sweeps):
    case = cases('C2', frames=200)
    labels = list(case['latent_labels'])
    M = len(labels)
    folds = [[2], [4, M - 1], [M // 2]]
    cfg = case['cfg']
    cap = chmosh._read_capture(case['mocap_fname'], cfg, labels, 'general', True)
    assert cap['raw_cols'] is not None
    sub = chmosh._subject([cap], cfg, case['markers_latent'], labels, case['betas'], case['marker_meta'], None, 0)
    hide = np.zeros((len(folds), M), dtype=bool)
    for k, f in enumerate(folds):
        hide[k, f] = True
    sched = chmosh._resolve_schedule(sub['pk'], 'fast', [cap['F']] * len(folds), None, None, None, None, None, True, None, chmosh.NUM_SMS)
    assert sched['chunk_len'] > 0
    out, _ = chmosh._solve_launch([dict(sub, seqs=[cap] * len(folds))], sched, time.time(), sequence_sweeps=sweeps, folds=hide,
                                  fold_rows=True)
    fns = []
    for k, f in enumerate(folds):
        fn, _ = capture_with(case, tmp_path, f'fold{k}_{sweeps}', lambda mk, L, f=f: mk.__setitem__(
            (slice(None), [L.index(labels[i]) for i in f]), np.nan))
        fns.append(fn)
    batch = chmosh.mosh_stageii_batch(fns, cfg, case['markers_latent'], labels, case['betas'], case['marker_meta'],
                                      sequence_sweeps=sweeps)
    F, rows = cap['F'], out['rows']
    for k, b in enumerate(batch):
        r = chmosh._SeqResult(rows, k * F, (k + 1) * F)
        bb = b['stageii_debug_details']['b200']
        ok = (r.status & lib.ST_SOLVED) != 0
        assert np.array_equal(np.flatnonzero(ok), bb['frame_ids'])
        assert r.pose[ok].tobytes() == bb['pose_reduced'].tobytes()
        assert r.fullpose[ok].tobytes() == b['fullpose'].tobytes() and r.trans[ok].tobytes() == b['trans'].tobytes()
        assert np.array_equal(out['status'][k], bb['status'])
    # the device errors are those of the fold rows
    obs, vis = cap['mocap'].frames_for_labels(labels, cap['sel'])
    for k, f in enumerate(folds):
        sim = rows.markers_sim[k * F:(k + 1) * F][:, f]
        e = np.linalg.norm(sim - obs[:, f], axis=-1)
        e[~vis[:, f] | ((out['status'][k] & lib.ST_SOLVED) == 0)[:, None]] = np.nan
        assert np.array_equal(np.isnan(e), np.isnan(out['err'][k][:, :len(f)]))
        assert np.nanmax(np.abs(e - out['err'][k][:, :len(f)])) < 1e-12


# Behaviour: a latent marker of the Stage-I output shifted by 3 cm must stand out.  Held-out means differ between markers by
# more than that on their own (BASELINE.md section 5: on this capture one marker's held-out mean is above 10 cm), so the shift is
# measured against the same call with the Stage-I output as it is: the shifted label's mean must rise the most, by more than
# SHIFT_MARGIN times the largest change of any other label's mean.
SHIFT_MARGIN = 2.0


@pytest.mark.gpu
def test_gpu_shifted_latent_marker_stands_out(cases):
    case = cases('C2', frames=120)
    labels = list(case['latent_labels'])
    i = len(labels) // 3
    ml = np.array(case['markers_latent'], dtype=np.float64)
    ml[i] += np.array([0.03, 0.0, 0.0])
    means = []
    for latent in (case['markers_latent'], ml):
        out = chmosh.mosh_stageii(case['mocap_fname'], case['cfg'], latent, labels, case['betas'], case['marker_meta'], heldout='each',
                                  subject_cache=False)
        means.append({l: s['mean'] for l, s in out['stageii_debug_details']['b200']['heldout']['per_label'].items()})
    rise = {l: means[1][l] - means[0][l] for l in means[0]}
    others = max(abs(v) for l, v in rise.items() if l != labels[i])
    print(f'shifted {labels[i]}: held-out mean {means[0][labels[i]] * 1e3:.2f} -> {means[1][labels[i]] * 1e3:.2f} mm; largest change of '
          f'another label {others * 1e3:.2f} mm (ratio {rise[labels[i]] / others:.1f}); largest held-out mean of the clean run '
          f'{max(means[0].values()) * 1e3:.2f} mm ({max(means[0], key=means[0].get)})')
    assert max(rise, key=rise.get) == labels[i]
    assert rise[labels[i]] > SHIFT_MARGIN * others
