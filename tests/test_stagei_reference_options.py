"""Stage I with ``mosh_stagei(..., reference_options=True)``: the head-marker correlation prior (``moshpp.head_marker_corr_fname``,
reference chmosh.py:252-266,360-373) and the extra initial rigid adjustment (``opt_settings.extra_initial_rigid_adjustment``,
chmosh.py:230-232), as the reference runs them.

The float64 oracle is ``oracle.stagei`` with ``reference_options=True``:
  - the init terms: every type other than 'head' covers its markers minus the correlated ones, the 'head' type is dropped,
    and ``init_head_corr = corr (ml - init)[head_ids] * wt`` with wt the 'body' type's init weight, else the base one;
  - after the per-frame rigid fit, one dog-leg over the unweighted data residual wrt every frame's root orientation and
    translation (e_3 = 1e-3, delta_0 = 0.5, maxiter), the rest fixed.

CPU: the oracle's new rows against finite differences; the product on the host build of the device source against the oracle
(C2 with the prior, a layout with 'head'-type markers, CF with the rigid adjustment, CF with a free shape and both options);
the availability rule, the keyword's default and the reported terms; the head end to end.  `-m gpu`: the CUDA library against
the oracle, and its result feeding Stage II."""
import copy
import functools
import json
import os
import pickle
import shutil

import numpy as np
import pytest

from conftest import EmuStageIBackend, stagei_case
from moshpp_b200 import stagei as product
from oracle import stagei as oracle
from test_stagei import _compare as _compare_body
from test_stagei_face import _compare as _compare_face, face_case

HEAD = ['LFHD', 'RFHD', 'LBHD', 'RBHD']


def write_corr(fname, labels, extra_rows=2, seed=0):
    """A head-marker correlation file: ``mrk_labels`` (H) and ``corr`` (K x H, K = H + extra_rows)."""
    rng = np.random.default_rng(seed)
    H = len(labels)
    corr = np.vstack([np.eye(H) + rng.normal(0, 0.2, (H, H)), rng.normal(0, 0.5, (extra_rows, H))])
    np.savez(fname, mrk_labels=np.asarray(labels), corr=corr)
    return fname


def relabel(meta, types):
    """A copy of a marker layout with some labels moved to other types ({label: type}); the masks follow."""
    meta = copy.deepcopy(meta)
    labels = list(meta['marker_vids'])
    for l, t in types.items():
        meta['marker_type'][l] = t
        meta['m2b_distance'].setdefault(t, 0.0095)
    names = sorted(set(meta['marker_type'].values()))
    meta['marker_type_mask'] = {t: np.array([meta['marker_type'][l] == t for l in labels]) for t in names}
    meta['m2b_distance'] = {t: meta['m2b_distance'][t] for t in names}
    return meta


def body_case(cases, tmp_path, n_pick=4):
    case, cfg, frames = stagei_case(cases, 'C2', n_pick, frames=40, n_verts=1500, dropout=0.02)
    assert all(l in case['marker_meta']['marker_vids'] for l in HEAD)
    cfg.moshpp.head_marker_corr_fname = write_corr(str(tmp_path / 'head_corr.npz'), HEAD)
    return case, cfg, frames


def _check_stats(out, ref, n_min):
    st, rs = out['stagei_debug_details']['b200'], ref['stagei_debug_details']['oracle_stats']
    assert st['linearisations'] == rs['j_evals'] and st['iterations'] == rs['iterations']
    assert st['minimisations'] == rs['minimizations'] == n_min


def _assert_bit_identical(a, b):
    assert np.array_equal(a['betas'], b['betas']) and np.array_equal(a['markers_latent'], b['markers_latent'])
    da, db = a['stagei_debug_details'], b['stagei_debug_details']
    for key in ('opt_models_pose', 'opt_models_trans', 'stagei_markers_sim_all'):
        assert all(np.array_equal(x, y) for x, y in zip(da[key], db[key])), key
    assert da['stagei_errs'] == db['stagei_errs'] and da['b200'] == db['b200']


def _emu(frames, cfg, meta, **kw):
    return product.mosh_stagei(frames, cfg, marker_meta=meta, backend=EmuStageIBackend(), **kw)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the oracle against finite differences
# ---------------------------------------------------------------------------------------------------------------------
def _fd_check(f, x0, J, cols, rows, h, tol):
    for c in cols:
        xp, xm = x0.copy(), x0.copy()
        xp[c] += h
        xm[c] -= h
        fd = (f(xp) - f(xm)) / (2 * h)
        assert np.abs(J[rows, c]).max() > 0, c
        assert np.abs(fd[rows] - J[rows, c]).max() < tol * np.abs(J[rows, c]).max(), c


def test_oracle_new_rows_equal_finite_differences(cases, tmp_path):
    """The init rows with the correlated markers left out and the init_head_corr rows (wrt the shape and the latent markers),
    and the rows of the extra rigid adjustment (wrt every frame's translation and root orientation)."""
    case, cfg, frames = stagei_case(cases, 'C2', 3, frames=40, n_verts=1500, dropout=0.0)
    cfg.moshpp.head_marker_corr_fname = write_corr(str(tmp_path / 'head_corr.npz'), HEAD)
    cfg.opt_settings.extra_initial_rigid_adjustment = True
    s = oracle.StageISolver(frames, cfg, case['marker_meta'], reference_options=True)
    s.rigid_adjust()
    wts = s.weights_for(0.5)
    pose_ids = s.pose_ids_for(True)
    rng = np.random.default_rng(0)
    x0 = s.get_x(pose_ids, True)
    nb, M = s.nb, s.n_markers
    ids = np.arange(len(x0))
    x0 = x0 + rng.normal(0, 0.02, x0.shape) * (ids >= nb + 3 * M) + rng.normal(0, 0.3, x0.shape) * (ids < nb)
    at = {}
    r, J = s.residual(x0, True, pose_ids, True, wts, True, rows=at)
    n_new = 3 * (M - len(HEAD)) + 3 * (len(HEAD) + 2)                     # init rows of the other markers + K x 3 corr rows
    rows = np.concatenate([np.arange(len(r))[sl] for k, sl in at.items() if k.startswith('init_')])     # init_head_corr last
    assert len(rows) == n_new
    h0, h1 = s.corr_ids[0], s.corr_ids[3]
    body = s.latent_labels.index('C7')
    cols = [0, 3, nb - 1, nb + 3 * h0, nb + 3 * h1 + 2, nb + 3 * body + 1]
    _fd_check(lambda x: s.residual(x, False, pose_ids, True, wts, True), x0, J, cols, rows, 1e-5, 5e-8)
    # the head rows couple the correlated markers densely, the other init rows do not see them
    assert np.count_nonzero(J[rows[-3 * (len(HEAD) + 2):], nb:nb + 3 * M].any(0)) == 3 * len(HEAD)
    assert not J[rows[:-3 * (len(HEAD) + 2)]][:, [nb + 3 * i + c for i in s.corr_ids for c in range(3)]].any()

    xr = np.hstack([s.trans, s.pose[:, :3]]).reshape(-1) + rng.normal(0, 0.02, 6 * s.n_frames)
    r, J = s.rigid_residual(xr, True)
    data = np.arange(3 * sum(len(i) for i in s.lm_ids))
    assert J.shape == (len(r), 6 * s.n_frames) and not r[len(data):].any() and not J[len(data):].any()
    _fd_check(lambda x: s.rigid_residual(x, False), xr, J, [0, 2, 3, 5, 6 + 4, 12 + 1], data, 1e-6, 5e-8)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the product on the host build of the device source against the oracle
# ---------------------------------------------------------------------------------------------------------------------
def test_head_corr_on_device_source_equals_oracle(cases, tmp_path):
    """1. C2 (SMPL-H, free shape, fingers), the correlated markers of type 'body'."""
    case, cfg, frames = body_case(cases, tmp_path)
    cfg.opt_settings.maxiter = 6
    meta = case['marker_meta']
    ref = oracle.mosh_stagei(frames, cfg, marker_meta=meta, reference_options=True)
    out = _emu(frames, cfg, meta, reference_options=True)
    _compare_body(out, ref, 1e-9)
    _check_stats(out, ref, 4)
    e = out['stagei_debug_details']['stagei_errs']
    assert e['init_head_corr'] > 0 and e['init_body'] > 0 and 'init_head' not in e


def test_head_typed_markers_on_device_source_equal_oracle(cases, tmp_path):
    """2. Two correlated labels of type 'head', two of type 'body', and a 'head' marker that is not in the file: that marker
    has no init term."""
    case, cfg, frames = body_case(cases, tmp_path)
    cfg.opt_settings.maxiter = 6
    meta = relabel(case['marker_meta'], {'LFHD': 'head', 'RFHD': 'head', 'ARIEL': 'head'})
    ref = oracle.mosh_stagei(frames, cfg, marker_meta=meta, reference_options=True)
    out = _emu(frames, cfg, meta, reference_options=True)
    _compare_body(out, ref, 1e-9)
    _check_stats(out, ref, 4)
    assert 'init_head' not in out['stagei_debug_details']['stagei_errs']
    # moving ARIEL's latent marker changes no init term (the data and surface terms do see it)
    s = product.StageI(frames, cfg, meta, backend=EmuStageIBackend(), reference_options=True)
    wts = s.weights_for(1.0)
    _, e0, _ = s.evaluate(False, wts, False)
    s.ml[s.labels.index('ARIEL')] += 0.01
    _, e1, _ = s.evaluate(False, wts, False)
    assert all(e0[k] == e1[k] for k in e0 if k.startswith('init_')) and e0['surf'] != e1['surf']
    s.ml[s.labels.index('RFHD')] += 0.01
    _, e2, _ = s.evaluate(False, wts, False)
    assert e2['init_head_corr'] != e1['init_head_corr'] and e2['init_body'] == e1['init_body']


def test_extra_rigid_adjustment_on_device_source_equals_oracle(cases, tmp_path):
    """3. CF (SMPL-X with face markers, the shape given) with the extra rigid adjustment: five minimisations."""
    case, cfg, frames, fn = face_case(cases, tmp_path)
    cfg.opt_settings.maxiter = 6
    cfg.opt_settings.extra_initial_rigid_adjustment = True
    meta = case['marker_meta']
    ref = oracle.mosh_stagei(frames, cfg, betas_fname=fn, marker_meta=meta, reference_options=True)
    out = _emu(frames, cfg, meta, betas_fname=fn, reference_options=True)
    _compare_face(out, ref, 1e-9)
    _check_stats(out, ref, 5)
    assert 'init_head_corr' not in out['stagei_debug_details']['stagei_errs']


def test_both_options_with_free_shape_face_on_device_source_equal_oracle(cases, tmp_path):
    """4. CF with a free shape and the face (face_with_free_shape) and both options."""
    case, cfg, frames = stagei_case(cases, 'CF', 4, frames=40, dropout=0.02)
    cfg.opt_settings.maxiter = 6
    cfg.opt_settings.extra_initial_rigid_adjustment = True
    cfg.moshpp.head_marker_corr_fname = write_corr(str(tmp_path / 'head_corr.npz'), HEAD, seed=1)
    meta = case['marker_meta']
    ref = oracle.mosh_stagei(frames, cfg, marker_meta=meta, face_with_free_shape=True, reference_options=True)
    out = _emu(frames, cfg, meta, face_with_free_shape=True, reference_options=True)
    _compare_face(out, ref, 1e-9)
    _check_stats(out, ref, 5)
    assert out['stagei_debug_details']['stagei_errs']['init_head_corr'] > 0


def test_head_corr_needs_every_label_in_the_layout(cases, tmp_path):
    """5. A file that names a label the layout does not have: the prior is skipped, bit for bit."""
    case, cfg, frames = body_case(cases, tmp_path, 3)
    cfg.opt_settings.maxiter = 2
    meta = case['marker_meta']
    cfg.moshpp.head_marker_corr_fname = write_corr(str(tmp_path / 'absent.npz'), HEAD[:3] + ['NOT_IN_LAYOUT'])
    a = _emu(frames, cfg, meta, reference_options=True)
    c = copy.deepcopy(cfg)
    c.moshpp.head_marker_corr_fname = None
    b = _emu(frames, c, meta, reference_options=True)
    _assert_bit_identical(a, b)
    assert 'init_head_corr' not in a['stagei_debug_details']['stagei_errs']


def test_options_off_in_cfg_keep_the_default_result(cases):
    """6. Both options off in cfg: reference_options=True gives the default's result, bit for bit."""
    case, cfg, frames = stagei_case(cases, 'C2', 3, frames=40, n_verts=1500, dropout=0.02)
    cfg.opt_settings.maxiter = 2
    cfg.moshpp.head_marker_corr_fname = None
    cfg.opt_settings.extra_initial_rigid_adjustment = False
    _assert_bit_identical(_emu(frames, cfg, case['marker_meta'], reference_options=True), _emu(frames, cfg, case['marker_meta']))


def test_missing_corr_file_raises(cases, tmp_path):
    """7. As in the reference, np.load of a missing file raises FileNotFoundError; without the keyword NotImplementedError."""
    case, cfg, frames = stagei_case(cases, 'C2', 3, frames=40, n_verts=1500, dropout=0.02)
    cfg.moshpp.head_marker_corr_fname = str(tmp_path / 'missing.npz')
    with pytest.raises(FileNotFoundError):
        _emu(frames, cfg, case['marker_meta'], reference_options=True)
    with pytest.raises(NotImplementedError, match='reference_options'):
        _emu(frames, cfg, case['marker_meta'])


def test_reported_init_terms(cases, tmp_path):
    """8. init_head_corr is reported, init_head is not, and a type whose markers are all correlated reports 0."""
    case, cfg, frames = body_case(cases, tmp_path, 3)
    meta = relabel(case['marker_meta'], dict({l: 'headband' for l in HEAD}, ARIEL='head'))
    s = product.StageI(frames, cfg, meta, backend=EmuStageIBackend(), reference_options=True)
    move = np.random.default_rng(2).normal(0, 0.005, s.ml.shape)           # (the latent markers start on their init)
    s.ml += move
    _, e, _ = s.evaluate(False, s.weights_for(1.0), False)
    assert e['init_head_corr'] > 0 and 'init_head' not in e
    assert e['init_headband'] == 0.0 and e['init_body'] > 0
    assert {k for k in e if k.startswith('init_')} == {'init_body', 'init_finger_left', 'init_finger_right', 'init_headband',
                                                       'init_head_corr'}
    o = oracle.StageISolver(frames, cfg, meta, reference_options=True)
    o.ml += move
    terms = {}
    o.residual(o.get_x(o.pose_ids_for(False), True), False, o.pose_ids_for(False), True, o.weights_for(1.0), False, terms)
    assert {k for k in terms if k.startswith('init_')} == {k for k in e if k.startswith('init_')}
    for k in ('init_head_corr', 'init_body', 'init_headband'):
        assert abs(terms[k] - e[k]) <= 1e-9 * abs(e[k]), k


def test_head_corr_weight_follows_the_body_type(cases, tmp_path):
    """9. The weight of init_head_corr is the 'body' type's init weight (stagei_wt_init_body when given), annealed, or the
    base weight when the layout has no 'body' type."""
    case, cfg, frames = body_case(cases, tmp_path, 3)
    w = cfg.opt_settings.weights
    w['stagei_wt_init_body'] = 3.0 * w['stagei_wt_init']
    meta = case['marker_meta']
    move = np.random.default_rng(3).normal(0, 0.005, (len(meta['marker_vids']), 3))
    s = product.StageI(frames, cfg, meta, backend=EmuStageIBackend(), reference_options=True)
    s.ml += move
    assert s.weights_for(0.5)['init_head_corr'] == 0.5 * w['stagei_wt_init_body'] == s.weights_for(0.5)['init']['body']
    _, e3, _ = s.evaluate(False, s.weights_for(0.5), False)
    c = copy.deepcopy(cfg)
    del c.opt_settings.weights['stagei_wt_init_body']
    s1 = product.StageI(frames, c, meta, backend=EmuStageIBackend(), reference_options=True)
    s1.ml += move
    _, e1, _ = s1.evaluate(False, s1.weights_for(0.5), False)
    assert e1['init_head_corr'] > 0 and np.isclose(e3['init_head_corr'], 9.0 * e1['init_head_corr'], rtol=1e-12)
    nobody = relabel(meta, {l: 'core' for l, t in meta['marker_type'].items() if t == 'body'})
    s2 = product.StageI(frames, cfg, nobody, backend=EmuStageIBackend(), reference_options=True)
    s2.ml += move
    assert 'body' not in s2.weights_for(0.5)['init']
    assert s2.weights_for(0.5)['init_head_corr'] == 0.5 * w['stagei_wt_init']
    _, e2, _ = s2.evaluate(False, s2.weights_for(0.5), False)
    assert np.isclose(e2['init_head_corr'], e1['init_head_corr'], rtol=1e-12)


def test_head_end_to_end_with_the_default_corr_path(tmp_path):
    """10. run_moshpp_once with the keyword bound and a correlation file at the cfg's derived path
    (<support_base_dir>/ssm_head_marker_corr.npz): the Stage-I pickle reports init_head_corr."""
    from moshpp_b200 import mosh_head, synth
    from oracle import stageii as oracle_stageii

    def stageii(mocap_fname, cfg, markers_latent, latent_labels, betas, marker_meta, v_template_fname=None):
        out = oracle_stageii.mosh_stageii(mocap_fname, cfg, markers_latent, latent_labels, betas, marker_meta, v_template_fname)
        out.pop('_pose_reduced')
        out['stageii_debug_details'].pop('oracle_stats')
        return out
    root = str(tmp_path)
    session = os.path.join(root, 'mocap', 'Synth DS', 'subject 01')
    os.makedirs(session)
    case = synth.make_case(os.path.join(root, 'models'), 'C2', frames=10, n_verts=1500)
    cap = os.path.join(session, 'take_00.npz')
    shutil.move(case['mocap_fname'], cap)
    with open(os.path.join(session, 'settings.json'), 'w') as f:
        json.dump({'gender': 'male'}, f)
    support = os.path.join(root, 'support')
    os.makedirs(support)
    write_corr(os.path.join(support, 'ssm_head_marker_corr.npz'), HEAD)
    sm = case['cfg'].surface_model
    cfg = {'mocap.fname': cap, 'dirs.work_base_dir': os.path.join(root, 'work'), 'dirs.support_base_dir': support,
           'surface_model.type': 'smplh', 'surface_model.fname': sm.fname,
           'moshpp.pose_body_prior_fname': case['cfg'].moshpp.pose_body_prior_fname,
           'moshpp.pose_hand_prior_fname': case['cfg'].moshpp.pose_hand_prior_fname, 'moshpp.optimize_fingers': True,
           'moshpp.stagei_frame_picker.num_frames': 4, 'moshpp.stagei_frame_picker.least_avail_markers': 0.8,
           'opt_settings.maxiter': 3}
    layout = os.path.join(root, 'work', 'SynthDS', 'SynthDS_smplh.json')
    os.makedirs(os.path.dirname(layout))
    product.write_marker_layout(layout, case['marker_meta'])
    np.random.seed(0)
    mp = mosh_head.run_moshpp_once(cfg, stagei_func=functools.partial(product.mosh_stagei, backend=EmuStageIBackend(),
                                                                      reference_options=True), stageii_func=stageii)
    assert mp.cfg.moshpp.head_marker_corr_fname == os.path.join(support, 'ssm_head_marker_corr.npz')
    with open(mp.stagei_fname, 'rb') as f:
        s1 = pickle.load(f)
    e = s1['stagei_debug_details']['stagei_errs']
    assert e['init_head_corr'] > 0 and 'init_head' not in e
    assert os.path.exists(mp.stageii_fname)


# ---------------------------------------------------------------------------------------------------------------------
# the CUDA path
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_head_corr_on_the_gpu_equals_oracle(cases, tmp_path):
    case, cfg, frames = body_case(cases, tmp_path)
    cfg.opt_settings.maxiter = 12
    meta = case['marker_meta']
    ref = oracle.mosh_stagei(frames, cfg, marker_meta=meta, reference_options=True)
    out = product.mosh_stagei(frames, cfg, marker_meta=meta, reference_options=True)
    _compare_body(out, ref, 1e-6)
    assert out['stagei_debug_details']['stagei_errs']['init_head_corr'] > 0


@pytest.mark.gpu
def test_extra_rigid_adjustment_on_the_gpu_equals_oracle(cases, tmp_path):
    case, cfg, frames, fn = face_case(cases, tmp_path)
    cfg.opt_settings.maxiter = 12
    cfg.opt_settings.extra_initial_rigid_adjustment = True
    meta = case['marker_meta']
    ref = oracle.mosh_stagei(frames, cfg, betas_fname=fn, marker_meta=meta, reference_options=True)
    out = product.mosh_stagei(frames, cfg, betas_fname=fn, marker_meta=meta, reference_options=True)
    _compare_face(out, ref, 1e-6)
    assert out['stagei_debug_details']['b200']['minimisations'] == 5


@pytest.mark.gpu
def test_both_options_with_free_shape_face_feed_stageii(cases, tmp_path):
    """Case 4 on the GPU, its result through Stage II (the library, optimize_face) on the CF sequence."""
    from moshpp_b200.chmosh import mosh_stageii
    case, cfg, frames = stagei_case(cases, 'CF', 4, frames=40, dropout=0.02)
    cfg.opt_settings.maxiter = 6
    cfg.opt_settings.extra_initial_rigid_adjustment = True
    cfg.moshpp.head_marker_corr_fname = write_corr(str(tmp_path / 'head_corr.npz'), HEAD, seed=1)
    si = product.mosh_stagei(frames, cfg, marker_meta=case['marker_meta'], face_with_free_shape=True, reference_options=True)
    assert si['stagei_debug_details']['b200']['minimisations'] == 5
    assert si['stagei_debug_details']['stagei_errs']['init_head_corr'] > 0
    out = mosh_stageii(mocap_fname=case['mocap_fname'], cfg=case['cfg'], precision='f64', chunk_len=0,
                       markers_latent=si['markers_latent'], latent_labels=si['latent_labels'], betas=si['betas'],
                       marker_meta=si['marker_meta'])
    assert out['fullpose'].shape[0] == out['expression'].shape[0] > 0
    assert np.isfinite(out['fullpose']).all() and np.isfinite(out['trans']).all() and np.isfinite(out['expression']).all()
