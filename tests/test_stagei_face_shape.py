"""Stage I on SMPL-X with face markers and a free shape (``mosh_stagei(..., face_with_free_shape=True)``): the shape and every
picked frame's jaw and expressions fitted together.  The reference refuses this case (chmosh.py:103-118,287-291) and suggests
two Stage-I runs instead; here it is the union of the free-shape objective and the face objective.

The float64 oracle is ``oracle.stagei`` with ``face_with_free_shape=True``: the data rows of a frame are posed on the frame's
own betas (the shape plus its expressions), and their columns wrt the shape come through both the frame's model and the
marker attachment on the canonical body (zero expressions).

CPU: the oracle against finite differences, the product on the host build of the device source against the oracle, the rules
that turn the face off, and the workspace plans at the reference's size.  `-m gpu`: the CUDA library against the oracle at CF
size and at 80 expressions, the joint fit against the two-pass procedure on a synthetic subject, and the MoSh head end to end.
"""
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
from moshpp_b200 import synth
from oracle import stagei as oracle
from test_face_reference_size import _NoBackend, _assert_plans, _relayout, emu_plan, face80_case  # noqa: F401 (emu_plan: a fixture)
from test_stagei_face import _assert_same_result, _compare, _face_labels


def joint_case(cases, n_pick=4, frames=40, **kw):
    """CF (SMPL-X with face markers, expressions moving in every frame) with optimize_betas and optimize_face."""
    case, cfg, frames = stagei_case(cases, 'CF', n_pick, frames=frames, dropout=0.02, **kw)
    assert cfg.moshpp.optimize_betas and cfg.moshpp.optimize_face
    return case, cfg, frames


def _check_joint_result(out, cfg, n_expr):
    nb = cfg.surface_model.num_betas
    do = out['stagei_debug_details']
    assert np.abs(out['betas'][:nb]).max() > 1e-2 and not np.any(out['betas'][nb:])      # the shape moved; no expressions in it
    assert {'beta', 'poseF', 'expr'} <= set(do['stagei_errs']) and do['stagei_errs']['expr'] > 0
    assert np.stack(do['opt_models_expression']).shape == (len(do['opt_models_pose']), n_expr)
    assert np.abs(np.stack(do['opt_models_expression'])).max() > 1e-3                       # the expressions moved
    assert np.abs(np.stack(do['opt_models_pose'])[:, 66:69]).max() > 1e-3                   # the jaw moved
    assert not np.any(np.stack(do['opt_models_pose'])[:, 69:75])                             # the eyes did not


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the oracle, the host build of the device source, the rules, the workspace plans
# ---------------------------------------------------------------------------------------------------------------------
def test_joint_oracle_jacobian_equals_finite_differences(cases):
    case, cfg, frames = joint_case(cases, 3)
    s = oracle.StageISolver(frames, cfg, case['marker_meta'], face_with_free_shape=True)
    s.rigid_adjust()
    wts = s.weights_for(0.25)
    pose_ids = s.pose_ids_for(True)
    _, off_ml, off_fr, per, n = s.layout(pose_ids, True, True)
    per0 = s.layout(pose_ids, True)[3]
    nb, npi = s.nb, len(pose_ids)
    assert off_ml == nb == 16 and per == per0 + 8 and n == off_fr + 3 * per
    rng = np.random.default_rng(0)
    x0 = s.get_x(pose_ids, True, True)
    ids = np.arange(len(x0))
    frame_part = ids >= off_fr
    is_expr = frame_part & ((ids - off_fr) % per >= 3 + npi)
    x0 = (x0 + rng.normal(0, 0.02, x0.shape) * (frame_part & ~is_expr) + rng.normal(0, 0.5, x0.shape) * is_expr
          + rng.normal(0, 0.3, x0.shape) * (ids < nb))                                      # non-zero shape and expressions
    rows = {}
    r, J = s.residual(x0, True, pose_ids, True, wts, True, free_expr=True, rows=rows)
    assert J.shape == (len(r), n)
    jaw = int(np.nonzero(pose_ids == 66)[0][0])
    face_marker = s.latent_labels.index(_face_labels(case['marker_meta'])[3])
    cols = [0, 3, nb - 1,                                                                   # the shape
            off_fr + 3 + jaw, off_fr + per + 3 + jaw + 2,                                  # the jaw of frames 0 and 1
            off_fr + 3 + npi, off_fr + 3 + npi + 7, off_fr + per + 3 + npi + 2,               # expressions of frames 0 and 1
            off_ml + 3 * face_marker, off_ml + 3 * face_marker + 2,                           # one latent face marker
            off_fr + 2 * per + 1]                                                            # a translation

    def at(c, dx):
        x = x0.copy()
        x[c] += dx
        return s.residual(x, False, pose_ids, True, wts, True, free_expr=True)
    # the data rows of frames 0..2: their shape columns see the frame's expressions
    data = np.arange(len(r))[rows['data']]
    for c in cols:
        # (a small step: the surface distance of the latent face marker curves strongly, its O(h^2) error at h = 1e-6 is 1e-5;
        # the shape columns, large in the init and surface rows, take a larger one against rounding)
        h = 1e-7 if c >= nb else 1e-5
        fd = (at(c, h) - at(c, -h)) / (2 * h)
        assert np.abs(J[:, c]).max() > 0, c
        assert np.abs(fd - J[:, c]).max() < 1e-5 * (np.abs(J[:, c]).max() + 1e-9), c
        if c < nb:
            assert np.abs(J[data, c]).max() > 0 and np.abs(fd[data] - J[data, c]).max() < 5e-8 * np.abs(J[data, c]).max(), c


def test_joint_block_solve_on_device_source_equals_oracle(cases):
    """All four annealing steps: the shape in all, the jaw and the expressions in the last two; some frames miss markers."""
    case, cfg, frames = joint_case(cases)
    cfg.opt_settings.maxiter = 6
    meta = case['marker_meta']
    assert any(len(fr) < len(meta['marker_vids']) for fr in frames)
    ref = oracle.mosh_stagei(frames, cfg, marker_meta=meta, face_with_free_shape=True)
    out = product.mosh_stagei(frames, cfg, marker_meta=meta, backend=EmuStageIBackend(), face_with_free_shape=True)
    _compare(out, ref, 1e-9)
    st, rs = out['stagei_debug_details']['b200'], ref['stagei_debug_details']['oracle_stats']
    assert st['linearisations'] == rs['j_evals'] and st['iterations'] == rs['iterations'] and st['minimisations'] == 4
    _check_joint_result(out, cfg, 8)


def _flag_on_off(frames, cfg, meta):
    """With face_with_free_shape set, a case where a rule turns the face off gives plain free-shape Stage I."""
    runs = []
    for face in (True, False):
        c = copy.deepcopy(cfg)
        c.moshpp.optimize_face = face
        runs.append(product.mosh_stagei(frames, c, marker_meta=meta, backend=EmuStageIBackend(), face_with_free_shape=face))
    _assert_same_result(*runs)


def test_flag_with_face_marker_types_excluded_is_plain_free_shape(cases):
    """mocap.exclude_marker_types names the face: off before anything else looks at the layout, which here still has them."""
    case, cfg, frames = joint_case(cases, 3)
    cfg.opt_settings.maxiter = 2
    cfg.mocap.exclude_marker_types = ['face']
    assert _face_labels(case['marker_meta'])
    _flag_on_off(frames, cfg, case['marker_meta'])


def test_flag_without_face_markers_in_the_layout_is_plain_free_shape(cases, tmp_path):
    case, cfg, frames = joint_case(cases, 3)
    cfg.opt_settings.maxiter = 2
    layout = synth.write_marker_layout(str(tmp_path / 'layout.json'), case['marker_meta'])
    meta = product.load_marker_layout(layout, labels_map=None, exclude_marker_types=['face'])
    assert not _face_labels(meta)
    _flag_on_off(frames, cfg, meta)


def test_flag_without_face_labels_in_the_frames_is_plain_free_shape(cases):
    case, cfg, frames = joint_case(cases, 3)
    cfg.opt_settings.maxiter = 2
    face = set(_face_labels(case['marker_meta']))
    _flag_on_off([{l: v for l, v in fr.items() if l not in face} for fr in frames], cfg, case['marker_meta'])


def test_flag_on_smplh_is_plain_free_shape(cases):
    case, cfg, frames = stagei_case(cases, 'C2', 3, frames=40, n_verts=1500, dropout=0.02)
    cfg.opt_settings.maxiter = 2
    meta = copy.deepcopy(case['marker_meta'])
    labels = list(meta['marker_vids'])
    for l in labels[:4]:
        meta['marker_type'][l] = 'face'
    meta['m2b_distance']['face'] = 0.0095
    meta['marker_type_mask'] = {t: np.array([meta['marker_type'][l] == t for l in labels]) for t in meta['m2b_distance']}
    assert cfg.moshpp.optimize_betas and any(l in frames[0] for l in labels[:4])
    _flag_on_off(frames, cfg, meta)


def test_without_the_flag_smplx_face_with_free_shape_still_raises(cases):
    case, cfg, frames = joint_case(cases, 3)
    for kw in ({}, dict(face_with_free_shape=False)):
        with pytest.raises(NotImplementedError):
            product.mosh_stagei(frames, cfg, marker_meta=case['marker_meta'], backend=EmuStageIBackend(), **kw)
        with pytest.raises(NotImplementedError):
            product.StageI(frames, cfg, case['marker_meta'], backend=_NoBackend(), **kw)


def _joint80_pack(cases, n_markers):
    case = face80_case(cases)
    cfg = copy.deepcopy(case['cfg'])
    cfg.moshpp.optimize_fingers = True
    cfg.moshpp.optimize_betas = True
    labels, meta, _ = _relayout(case, n_markers)
    s = product.StageI([{l: np.zeros(3) for l in labels}], cfg, meta, backend=_NoBackend(), face_with_free_shape=True)
    assert s.face and s.free_betas and (s.nb, s.ne) == (16, 80)
    return s.pack_for(True)


@pytest.mark.parametrize('n_markers', [65, 90])
def test_joint80_workspace_plan_fits(cases, emu_plan, n_markers):  # noqa: F811
    """The reference's size: a linear block of 16 shape + 80 expression directions, Step 2 with 210 free variables (the
    jaw, 80 expressions, the fingers and 16 shape columns), both precisions, single- and multi-subject launches."""
    pk = _joint80_pack(cases, n_markers)
    assert (pk.n_dmpl, pk.n_expr, pk.n_markers) == (96, 80, n_markers)
    n1, n2 = len(pk.free_step1), len(pk.free_step2)
    assert n2 == 210 and list(pk.free_step2[-16:]) == [3 + pk.p_red + i for i in range(16)]
    assert list(pk.free_step2[n2 - 96:n2 - 16]) == [3 + pk.p_red + 16 + i for i in range(80)]
    assert list(pk.free_step1[n1 - 16:]) == [3 + pk.p_red + i for i in range(16)]
    _assert_plans(emu_plan, pk, ('SMPL-X-betas16-face80', n_markers, n2))
    for precision in ('f32', 'f64'):
        assert emu_plan(pk, precision, 0)['big'] == 1                                      # the global-workspace layout


# ---------------------------------------------------------------------------------------------------------------------
# the CUDA path
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_joint_stagei_on_the_gpu_equals_oracle(cases):
    """Per-frame linearisations from mosh2_job_linearize, closest points and distances from mosh2_mesh_distance."""
    case, cfg, frames = joint_case(cases)
    cfg.opt_settings.maxiter = 12
    ref = oracle.mosh_stagei(frames, cfg, marker_meta=case['marker_meta'], face_with_free_shape=True)
    out = product.mosh_stagei(frames, cfg, marker_meta=case['marker_meta'], face_with_free_shape=True)
    _compare(out, ref, 1e-6)
    _check_joint_result(out, cfg, 8)


@pytest.mark.gpu
def test_joint80_stagei_on_the_gpu_equals_oracle(cases):
    case, cfg, frames = joint_case(cases, 3, **synth.REFERENCE_FACE)
    cfg.opt_settings.maxiter = 4
    ref = oracle.mosh_stagei(frames, cfg, marker_meta=case['marker_meta'], face_with_free_shape=True)
    out = product.mosh_stagei(frames, cfg, marker_meta=case['marker_meta'], face_with_free_shape=True)
    _compare(out, ref, 1e-6)
    _check_joint_result(out, cfg, 80)


def _objective(frames, cfg, meta, res):
    """The joint Stage-I objective of the last annealing step at a result's state (shape, latent markers, poses,
    translations, expressions), evaluated by the library."""
    s = product.StageI(frames, cfg, meta, face_with_free_shape=True)
    s.betas[:] = res['betas']
    s.ml = res['markers_latent'].copy()
    dbg = res['stagei_debug_details']
    s.pose[:], s.trans[:], s.expr[:] = dbg['opt_models_pose'], dbg['opt_models_trans'], dbg['opt_models_expression']
    total, sse, _ = s.evaluate(False, s.weights_for(cfg.opt_settings.weights['stagei_wt_annealing'][-1]), True)
    return total, sse


@pytest.mark.gpu
def test_joint_fit_against_two_pass_on_ground_truth(cases, tmp_path):
    """A synthetic subject with known betas and expressions moving in every frame, fitted jointly and by the reference's
    recommended two passes: free shape with the face markers excluded, then the face with that shape given.  Both run to
    convergence (stagei_lr 1e-6): under the default relative-decrease stop (1e-3) the joint fit of this subject stops while
    the expressions are still near zero (on one H100: data SSE 9.9e3 against 3.2e3 for the two passes); converged it is the
    better fit (objective 2.53e3 against 2.96e3, data SSE 2.31e3 against 2.67e3, max beta error 0.87 against 1.30)."""
    case, cfg, frames = joint_case(cases, 12, frames=120)
    cfg.opt_settings.stagei_lr = 1e-6
    meta, nb = case['marker_meta'], cfg.surface_model.num_betas
    joint = product.mosh_stagei(frames, cfg, marker_meta=meta, face_with_free_shape=True)
    c1 = copy.deepcopy(cfg)
    c1.mocap.exclude_marker_types = ['face']
    layout = synth.write_marker_layout(str(tmp_path / 'layout.json'), meta)
    meta1 = product.load_marker_layout(layout, labels_map=None, exclude_marker_types=['face'])
    shape = product.mosh_stagei(frames, c1, marker_meta=meta1)
    fn = str(tmp_path / 'betas.npz')
    np.savez(fn, betas=shape['betas'])
    c2 = copy.deepcopy(cfg)
    c2.moshpp.optimize_betas = False
    two = product.mosh_stagei(frames, c2, betas_fname=fn, marker_meta=meta)
    report = {}
    for name, res in (('joint', joint), ('two_pass', two)):
        total, sse = _objective(frames, cfg, meta, res)
        report[name] = dict(beta_err=float(np.abs(res['betas'][:nb] - case['betas'][:nb]).max()), data_sse=sse['data'],
                            objective=total)
    print(json.dumps(report))
    assert report['joint']['objective'] <= report['two_pass']['objective']


@pytest.mark.gpu
def test_joint_stagei_through_the_head_feeds_stageii(tmp_path):
    """run_moshpp_once with the partial: the Stage-I pickle carries the fitted shape and every picked frame's expressions,
    and Stage II (the library, optimize_face) returns the expressions of the capture."""
    from moshpp_b200 import mosh_head
    root = str(tmp_path)
    session = os.path.join(root, 'mocap', 'Synth DS', 'subject 01')
    os.makedirs(session)
    case = synth.make_case(os.path.join(root, 'models'), 'CF', frames=60, n_verts=2000)
    cap = os.path.join(session, 'take_00.npz')
    shutil.move(case['mocap_fname'], cap)
    with open(os.path.join(session, 'settings.json'), 'w') as f:
        json.dump({'gender': 'male'}, f)
    sm = case['cfg'].surface_model
    cfg = {'mocap.fname': cap, 'dirs.work_base_dir': os.path.join(root, 'work'), 'dirs.support_base_dir': os.path.join(root, 'support'),
           'surface_model.type': 'smplx', 'surface_model.fname': sm.fname,
           'surface_model.betas_expr_start_id': sm.betas_expr_start_id, 'surface_model.num_expressions': sm.num_expressions,
           'moshpp.pose_body_prior_fname': case['cfg'].moshpp.pose_body_prior_fname,
           'moshpp.pose_hand_prior_fname': case['cfg'].moshpp.pose_hand_prior_fname, 'moshpp.optimize_fingers': True,
           'moshpp.optimize_face': True, 'moshpp.optimize_betas': True,
           'moshpp.stagei_frame_picker.num_frames': 4, 'moshpp.stagei_frame_picker.least_avail_markers': 0.8,
           'opt_settings.maxiter': 4, 'moshpp.head_marker_corr_fname': None}
    layout = os.path.join(root, 'work', 'SynthDS', 'SynthDS_smplx.json')
    os.makedirs(os.path.dirname(layout))
    product.write_marker_layout(layout, case['marker_meta'])
    np.random.seed(0)
    mp = mosh_head.run_moshpp_once(cfg, stagei_func=functools.partial(product.mosh_stagei, face_with_free_shape=True))
    with open(mp.stagei_fname, 'rb') as f:
        s1 = pickle.load(f)
    ex = np.stack(s1['stagei_debug_details']['opt_models_expression'])
    assert ex.shape == (4, 8) and np.abs(ex).max() > 1e-3
    assert np.abs(s1['betas'][:sm.num_betas]).max() > 1e-2
    with open(mp.stageii_fname, 'rb') as f:
        s2 = pickle.load(f)
    assert s2['expression'].shape[0] == s2['fullpose'].shape[0] == 60 and np.abs(s2['expression']).max() > 1e-3
