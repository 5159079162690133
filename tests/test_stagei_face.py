"""Stage I with ``optimize_face`` (reference chmosh.py:83-455): the jaw and the expression coefficients of every picked frame,
fitted with a given shape.  Each frame's model carries the given shape plus its own expressions; the jaw and the expressions
are free, with their poseF / expr terms, in the two detailed annealing steps only.  CPU: the oracle against finite
differences, and the product's block solve on the host build of the device source against the oracle.  `-m gpu`: the
CUDA library, alone and feeding Stage II.  The float64 oracle is ``oracle.stagei`` with the face on (``optimize_face`` and a
given shape)."""
import copy

import numpy as np
import pytest

from conftest import EmuStageIBackend, stagei_case
from moshpp_b200 import lib
from moshpp_b200 import stagei as product
from oracle import stagei as oracle

POSEF, EXPR = lib.ERR_NAMES.index('poseF'), lib.ERR_NAMES.index('expr')


def face_case(cases, tmp_path, n_pick=4):
    """CF (SMPL-X with face markers) with the shape given from a betas file and optimize_betas off."""
    case, cfg, frames = stagei_case(cases, 'CF', n_pick, frames=40, dropout=0.02)
    cfg.moshpp.optimize_betas = False
    fn = str(tmp_path / 'betas.npz')
    np.savez(fn, betas=case['betas'])
    return case, cfg, frames, fn


def _compare(out, ref, tol):
    assert np.abs(out['betas'] - ref['betas']).max() < tol
    assert np.abs(out['markers_latent'] - ref['markers_latent']).max() < tol
    do, dr = out['stagei_debug_details'], ref['stagei_debug_details']
    for key in ('opt_models_pose', 'opt_models_trans', 'opt_models_expression'):
        assert len(do[key]) == len(dr[key])
        for a, b in zip(do[key], dr[key]):
            assert a.shape == b.shape and np.abs(a - b).max() < tol, key
    assert set(do['stagei_errs'].keys()) == set(dr['stagei_errs'].keys()) >= {'poseF', 'expr'}
    for k, v in dr['stagei_errs'].items():
        assert abs(do['stagei_errs'][k] - v) <= 1e-5 * abs(v) + 100 * tol, k
    assert out['latent_labels'] == ref['latent_labels'] and out['markers_latent_vids'] == ref['markers_latent_vids']
    assert do['stagei_labels_obs'] == dr['stagei_labels_obs']
    for a, b in zip(do['stagei_markers_sim'], dr['stagei_markers_sim']):
        assert a.shape == b.shape and np.abs(a - b).max() < 10 * tol


def _assert_same_result(a, b):
    assert np.array_equal(a['betas'], b['betas']) and np.array_equal(a['markers_latent'], b['markers_latent'])
    da, db = a['stagei_debug_details'], b['stagei_debug_details']
    assert 'opt_models_expression' not in da and 'opt_models_expression' not in db
    for key in ('opt_models_pose', 'opt_models_trans', 'stagei_markers_sim_all'):
        assert all(np.array_equal(x, y) for x, y in zip(da[key], db[key])), key
    assert da['stagei_errs'] == db['stagei_errs'] and da['b200'] == db['b200']


def _face_labels(meta):
    return [l for l, t in meta['marker_type'].items() if 'face' in t]


def test_oracle_face_jacobian_equals_finite_differences(cases, tmp_path):
    case, cfg, frames, _ = face_case(cases, tmp_path, 3)
    s = oracle.StageISolver(frames, cfg, case['marker_meta'], case['betas'])
    assert len(s.expr_ids) == 8
    s.rigid_adjust()
    wts = s.weights_for(0.25)
    pose_ids = s.pose_ids_for(True)
    assert {66, 67, 68} <= set(pose_ids.tolist())
    _, off_ml, off_fr, per, n = s.layout(pose_ids, False, True)
    npi, M = len(pose_ids), s.n_markers
    rng = np.random.default_rng(0)
    x0 = s.get_x(pose_ids, False, True)
    ids = np.arange(len(x0))
    frame_part = ids >= off_fr
    is_expr = frame_part & ((ids - off_fr) % per >= 3 + npi)
    x0 = x0 + rng.normal(0, 0.02, x0.shape) * (frame_part & ~is_expr) + rng.normal(0, 0.5, x0.shape) * is_expr
    r, J = s.residual(x0, True, pose_ids, False, wts, True, free_expr=True)
    jaw = int(np.nonzero(pose_ids == 66)[0][0])
    face_marker = s.latent_labels.index(_face_labels(case['marker_meta'])[3])
    cols = [off_fr + 3 + jaw, off_fr + per + 3 + jaw + 2,                                  # the jaw of frames 0 and 1
            off_fr + 3 + npi, off_fr + 3 + npi + 7, off_fr + per + 3 + npi + 2,               # expressions of frames 0 and 1
            off_ml + 3 * face_marker, off_ml + 3 * face_marker + 2,                           # one latent face marker
            off_fr + 2 * per + 1]                                                            # a translation
    assert J.shape[1] == n == off_fr + 3 * per

    def at(c, dx):
        x = x0.copy()
        x[c] += dx
        return s.residual(x, False, pose_ids, False, wts, True, free_expr=True)
    for c in cols:
        # (a small step: the surface distance of the latent face marker curves strongly, its O(h^2) error at h = 1e-6 is 1e-5)
        h = 1e-7
        fd = (at(c, h) - at(c, -h)) / (2 * h)
        assert np.abs(J[:, c]).max() > 0, c
        assert np.abs(fd - J[:, c]).max() < 1e-5 * (np.abs(J[:, c]).max() + 1e-9), c


def test_face_block_solve_on_device_source_equals_oracle(cases, tmp_path):
    """All four annealing steps with the jaw and the expressions free in the last two; some picked frames miss markers."""
    case, cfg, frames, fn = face_case(cases, tmp_path)
    cfg.opt_settings.maxiter = 6
    meta = case['marker_meta']
    assert any(len(fr) < len(meta['marker_vids']) for fr in frames)
    ref = oracle.mosh_stagei(frames, cfg, betas_fname=fn, marker_meta=meta)
    out = product.mosh_stagei(frames, cfg, betas_fname=fn, marker_meta=meta, backend=EmuStageIBackend())
    _compare(out, ref, 1e-9)
    st, rs = out['stagei_debug_details']['b200'], ref['stagei_debug_details']['oracle_stats']
    assert st['linearisations'] == rs['j_evals'] and st['iterations'] == rs['iterations'] and st['minimisations'] == 4
    nb = cfg.surface_model.num_betas
    assert np.array_equal(out['betas'][:nb], case['betas'][:nb]) and not np.any(out['betas'][nb:])
    do = out['stagei_debug_details']
    assert 'beta' not in do['stagei_errs'] and do['stagei_errs']['expr'] > 0 and do['stagei_errs']['poseF'] > 0
    assert np.abs(np.stack(do['opt_models_expression'])).max() > 1e-3                      # the expressions moved
    assert np.abs(np.stack(do['opt_models_pose'])[:, 66:69]).max() > 1e-3                  # the jaw moved
    assert not np.any(np.stack(do['opt_models_pose'])[:, 69:75])                            # the eyes did not


def _linearize_face_weights(backend, cases, tmp_path):
    """One Step-2 linearisation at a state with a non-zero jaw and non-zero expressions: the poseF / expr SSE of every frame
    are the plain weighted sums of squares, also on a frame with missing markers (no visibility annealing in Stage I)."""
    case, cfg, frames, _ = face_case(cases, tmp_path)
    s = product.StageI(frames, cfg, case['marker_meta'], betas=case['betas'], backend=backend)
    assert s.face and s.ne == 8
    assert (~s.vis).any(axis=1).any() and s.vis.any(axis=1).all()
    rng = np.random.default_rng(3)
    s.pose[:, :3] = rng.normal(0, 0.1, (s.F, 3))
    s.pose[:, 66:69] = rng.normal(0, 0.2, (s.F, 3))
    s.expr[:] = rng.normal(0, 0.5, s.expr.shape)
    wts = s.weights_for(0.25)
    pk = s.pack_for(True, s.can(s.betas[:s.nb]))
    x = np.zeros((s.F, pk.nx))
    x[:, :3], x[:, 3:3 + pk.p_red], x[:, 3 + pk.p_red:] = s.trans, s.pose, s.expr
    opts = lib.make_options(None, optimize_fingers=True, optimize_face=True)
    opts.wt_data, opts.wt_poseB, opts.wt_poseH = wts['data'], wts['poseB'], wts['poseH']
    opts.wt_poseF, opts.wt_expr = wts['poseF'], wts['expr']
    assert opts.wt_annealing > 0
    dev = backend.linearize(pk, opts, s.obs, s.vis, x, 2, True)
    want_f = ((wts['poseF'] * s.pose[:, 66:69]) ** 2).sum(1)
    want_e = ((wts['expr'] * s.expr) ** 2).sum(1)
    assert np.allclose(dev['errs'][:, POSEF], want_f, rtol=1e-13, atol=0)
    assert np.allclose(dev['errs'][:, EXPR], want_e, rtol=1e-13, atol=0)


def test_linearise_mode_face_weights_on_device_source(cases, tmp_path):
    _linearize_face_weights(EmuStageIBackend(), cases, tmp_path)


@pytest.mark.gpu
def test_linearise_mode_face_weights_on_the_gpu(cases, tmp_path):
    _linearize_face_weights(product.DeviceBackend(), cases, tmp_path)


def test_face_with_free_shape_on_smplx_raises(cases):
    case, cfg, frames = stagei_case(cases, 'CF', 4, frames=40, dropout=0.02)
    assert cfg.moshpp.optimize_betas and cfg.moshpp.optimize_face
    with pytest.raises(NotImplementedError):
        product.mosh_stagei(frames, cfg, marker_meta=case['marker_meta'], backend=EmuStageIBackend())


def _on_off(frames, cfg, meta, fn=None):
    runs = []
    for face in (True, False):
        c = copy.deepcopy(cfg)
        c.moshpp.optimize_face = face
        runs.append(product.mosh_stagei(frames, c, betas_fname=fn, marker_meta=meta, backend=EmuStageIBackend()))
    _assert_same_result(*runs)


def test_face_without_face_markers_in_the_layout_is_off(cases, tmp_path):
    """No face-type marker in the layout (here with a free shape: the availability rule comes before the shape rule)."""
    from moshpp_b200 import synth
    case, cfg, frames = stagei_case(cases, 'CF', 3, frames=40, dropout=0.02)
    cfg.opt_settings.maxiter = 2
    layout = synth.write_marker_layout(str(tmp_path / 'layout.json'), case['marker_meta'])
    meta = product.load_marker_layout(layout, labels_map=None, exclude_marker_types=['face'])
    assert not _face_labels(meta) and len(meta['marker_vids']) < len(case['marker_meta']['marker_vids'])
    _on_off(frames, cfg, meta)


def test_face_without_face_labels_in_the_frames_is_off(cases, tmp_path):
    case, cfg, frames, fn = face_case(cases, tmp_path, 3)
    cfg.opt_settings.maxiter = 2
    face = set(_face_labels(case['marker_meta']))
    frames = [{l: v for l, v in fr.items() if l not in face} for fr in frames]
    _on_off(frames, cfg, case['marker_meta'], fn)


def test_face_on_smplh_is_ignored(cases):
    """Only SMPL-X has a jaw and expression components: on SMPL-H optimize_face changes nothing, even with markers of a face
    type in the layout and a free shape."""
    case, cfg, frames = stagei_case(cases, 'C2', 3, frames=40, n_verts=1500, dropout=0.02)
    cfg.opt_settings.maxiter = 2
    meta = copy.deepcopy(case['marker_meta'])
    labels = list(meta['marker_vids'])
    for l in labels[:4]:
        meta['marker_type'][l] = 'face'
    meta['m2b_distance']['face'] = 0.0095
    meta['marker_type_mask'] = {t: np.array([meta['marker_type'][l] == t for l in labels]) for t in meta['m2b_distance']}
    assert cfg.moshpp.optimize_betas and any(l in frames[0] for l in labels[:4])
    _on_off(frames, cfg, meta)


def test_other_stagei_options_still_raise(cases, tmp_path):
    case, cfg, frames, fn = face_case(cases, tmp_path, 3)
    c = copy.deepcopy(cfg)
    c.moshpp.head_marker_corr_fname = str(tmp_path / 'head_corr.npz')
    with pytest.raises(NotImplementedError):
        product.mosh_stagei(frames, c, betas_fname=fn, marker_meta=case['marker_meta'], backend=EmuStageIBackend())
    c = copy.deepcopy(cfg)
    c.opt_settings.extra_initial_rigid_adjustment = True
    with pytest.raises(NotImplementedError):
        product.mosh_stagei(frames, c, betas_fname=fn, marker_meta=case['marker_meta'], backend=EmuStageIBackend())


# ---------------------------------------------------------------------------------------------------------------------
# the CUDA path
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def gpu_face_stagei(cases, tmp_path_factory):
    import time
    case, cfg, frames, fn = face_case(cases, tmp_path_factory.mktemp('face'))
    cfg.opt_settings.maxiter = 12
    ref = oracle.mosh_stagei(frames, cfg, betas_fname=fn, marker_meta=case['marker_meta'])
    product.DeviceBackend()                 # (loads the library outside the timed call)
    t0 = time.perf_counter()
    out = product.mosh_stagei(frames, cfg, betas_fname=fn, marker_meta=case['marker_meta'])
    dt = time.perf_counter() - t0
    print(f'stage I with face on the GPU ({len(frames)} frames): {dt:.2f} s, {out["stagei_debug_details"]["b200"]}')
    return case, cfg, out, ref


@pytest.mark.gpu
def test_face_stagei_on_the_gpu_equals_oracle(gpu_face_stagei):
    """Per-frame linearisations from mosh2_job_linearize, closest points and distances from mosh2_mesh_distance."""
    case, cfg, out, ref = gpu_face_stagei
    _compare(out, ref, 1e-6)


@pytest.mark.gpu
def test_face_stagei_feeds_stageii(cases, gpu_face_stagei):
    """Stage I with face, then Stage II with face on a CF sequence: latent face markers, jaw and expressions end to end."""
    from moshpp_b200.chmosh import mosh_stageii
    from oracle import stageii
    _, _, si, _ = gpu_face_stagei
    case = cases('CF')
    assert si['latent_labels'] == case['latent_labels']
    args = dict(markers_latent=si['markers_latent'], latent_labels=si['latent_labels'], betas=si['betas'],
                marker_meta=si['marker_meta'])
    out = mosh_stageii(mocap_fname=case['mocap_fname'], cfg=case['cfg'], precision='f64', chunk_len=0, **args)
    ref = stageii.mosh_stageii(case['mocap_fname'], case['cfg'], args['markers_latent'], args['latent_labels'], args['betas'],
                               args['marker_meta'])
    assert out['expression'].shape == ref['expression'].shape
    assert np.abs(out['expression'] - ref['expression']).max() < 1e-8
    assert np.abs(out['fullpose'] - ref['fullpose']).max() < 1e-8
    assert np.abs(out['fullpose'][:, 66:69]).max() > 1e-3
    dbg, rdbg = out['stageii_debug_details'], ref['stageii_debug_details']
    assert set(dbg['stageii_errs'].keys()) == set(rdbg['stageii_errs'].keys()) >= {'poseF', 'expr'}
    for k in ('poseF', 'expr'):
        assert np.allclose(dbg['stageii_errs'][k], rdbg['stageii_errs'][k], rtol=1e-7, atol=1e-10)
