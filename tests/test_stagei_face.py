"""Stage I with ``optimize_face`` (reference chmosh.py:83-455): the jaw and the expression coefficients of every picked frame,
fitted with a given shape.  Each frame's model carries the given shape plus its own expressions; the jaw and the expressions
are free, with their poseF / expr terms, in the two detailed annealing steps only.  CPU: the oracle against finite
differences, and the product's block solve on the host build of the device source against the oracle.  `-m gpu`: the
CUDA library, alone and feeding Stage II.

The float64 oracle of the face objective, ``FaceOracle``, is built here on ``oracle/stagei.py``: the terms that do not see
the expressions (pose prior, init, surface, fingers) come from ``StageISolver.residual`` evaluated with no data rows; the
data term is restated with each frame's own betas and its columns wrt the expressions, and the poseF / expr terms are added."""
import copy

import numpy as np
import pytest
from sklearn.neighbors import NearestNeighbors

from conftest import EmuStageIBackend, stagei_case
from moshpp_b200 import lib
from moshpp_b200 import stagei as product
from oracle import stagei as oracle
from oracle.dogleg import minimize_dogleg
from oracle.lbs import LBS
from oracle.markers import TransformedCoeffs, transformed_lms

POSEF, EXPR = lib.ERR_NAMES.index('poseF'), lib.ERR_NAMES.index('expr')


class FaceOracle(oracle.StageISolver):
    """Stage I with optimize_face and a given shape (chmosh.py:136-151,163-170,283-295,322-324,396-401): every frame's model
    has its own betas, the given shape plus the frame's expressions at betas[betas_expr_start_id:][:num_expressions]; the
    canonical body keeps zero expressions.  In the detailed steps the jaw joins pose_ids and every frame's expressions are
    free, after its pose in the frame block: [trans | pose[pose_ids] | expressions]."""

    def __init__(self, stagei_frames, cfg, marker_meta, betas):
        super().__init__(stagei_frames, cfg, marker_meta, betas=betas)
        sm = cfg.surface_model
        assert sm.type == 'smplx' and not self.optimize_betas
        self.face_ids = [66, 67, 68]                                                            # the jaw
        es = int(sm.betas_expr_start_id)
        self.expr_ids = np.arange(es, es + int(sm.num_expressions))
        self.expr = np.zeros((self.n_frames, len(self.expr_ids)))

    def pose_ids_for(self, detailed):
        ids = super().pose_ids_for(detailed)
        return np.asarray(sorted(set(ids.tolist()) | set(self.face_ids)), dtype=np.int64) if detailed else ids

    def weights_for(self, anneal):
        out = super().weights_for(anneal)
        w = self.cfg.opt_settings.weights
        out['poseF'], out['expr'] = w['stagei_wt_poseF'] * anneal, w['stagei_wt_expr'] * anneal
        return out

    def frame_betas(self, f):
        b = self.betas.copy()
        b[self.expr_ids] = self.expr[f]
        return b

    def markers_sim_all(self, tc=None, can_v=None):
        can_v = self.can_v() if can_v is None else can_v
        tc = TransformedCoeffs(can_v, self.ml) if tc is None else tc
        lbs = LBS(self.model, tc.closest[:, :3].reshape(-1))
        out = []
        for f in range(self.n_frames):
            v = lbs(self.pose[f], self.frame_betas(f), self.trans[f]).reshape(-1, 3, 3)
            out.append(transformed_lms(tc, v[:, 0], v[:, 1], v[:, 2]))
        return out

    # ---- unknowns: the base layout (no free betas) with the free expressions appended to every frame block
    def face_layout(self, pose_ids, detailed):
        _, off_ml, off_fr, per0, _ = self.layout(pose_ids, False)
        per = per0 + (len(self.expr_ids) if detailed else 0)
        return off_ml, off_fr, per0, per, off_fr + self.n_frames * per

    def get_face_x(self, pose_ids, detailed):
        _, off_fr, per0, per, _ = self.face_layout(pose_ids, detailed)
        x0 = self.get_x(pose_ids, False)
        fr = np.hstack([x0[off_fr:].reshape(self.n_frames, per0), self.expr[:, :per - per0]])
        return np.concatenate([x0[:off_fr], fr.reshape(-1)])

    def set_face_x(self, x, pose_ids, detailed):
        _, off_fr, per0, per, _ = self.face_layout(pose_ids, detailed)
        fr = x[off_fr:].reshape(self.n_frames, per)
        self.expr[:, :per - per0] = fr[:, per0:]
        self.set_x(np.concatenate([x[:off_fr], fr[:, :per0].reshape(-1)]), pose_ids, False)

    def face_residual(self, x, want_jac, pose_ids, wts, detailed, per_term=None):
        self.set_face_x(x, pose_ids, detailed)
        off_ml, off_fr, per0, per, n = self.face_layout(pose_ids, detailed)
        M, F, npi = self.n_markers, self.n_frames, len(pose_ids)
        # the base class's terms with the data rows left out
        obs, lm_ids = self.obs, self.lm_ids
        self.obs, self.lm_ids = [o[:0] for o in obs], [i[:0] for i in lm_ids]
        try:
            base = self.residual(self.get_x(pose_ids, False), want_jac, pose_ids, False, wts, detailed, per_term)
        finally:
            self.obs, self.lm_ids = obs, lm_ids
        rs, Js = [base[0] if want_jac else base], []
        if want_jac:
            J0 = base[1]
            J = np.zeros((J0.shape[0], n))
            J[:, :off_fr] = J0[:, :off_fr]
            for f in range(F):
                J[:, off_fr + f * per:off_fr + f * per + per0] = J0[:, off_fr + f * per0:off_fr + (f + 1) * per0]
            Js.append(J)

        def block(name, r, J=None):
            rs.append(r)
            if per_term is not None:
                per_term[name] = per_term.get(name, 0.0) + float((r ** 2).sum())
            if want_jac:
                Js.append(J)

        # ---- data, posed on each frame's own model (its columns wrt the expressions: the posed vertices only)
        can_v = self.can_v()
        tc = TransformedCoeffs(can_v, self.ml)
        tri = tc.closest[:, :3]
        lbs = LBS(self.model, tri.reshape(-1))
        xids = self.expr_ids if detailed else self.expr_ids[:0]
        Fcan = np.stack([oracle.coeff_jacobians(can_v[tri[i]], self.ml[i])[1] for i in range(M)]) if want_jac else None
        for f in range(F):
            ids = self.lm_ids[f]
            res = lbs(self.pose[f], self.frame_betas(f), self.trans[f], want_jac, beta_ids=xids)
            verts = (res[0] if want_jac else res).reshape(M, 3, 3)
            if not want_jac:
                sim = transformed_lms(tc, verts[:, 0], verts[:, 1], verts[:, 2])
                block('data', ((self.obs[f] - sim[ids]) * wts['data']).reshape(-1))
                continue
            sim, loc = transformed_lms(tc, verts[:, 0], verts[:, 1], verts[:, 2], True)
            dv_pose = res[1].reshape(M, 3, 3, -1)
            dv_beta = res[2].reshape(M, 3, 3, -1)
            J = np.zeros((len(ids), 3, n))
            c0 = off_fr + f * per
            for row, i in enumerate(ids):
                e1, e2 = verts[i, 1] - verts[i, 0], verts[i, 2] - verts[i, 0]
                f1 = e1 / np.linalg.norm(e1)
                nn = np.cross(e1, e2)
                f2 = nn / np.linalg.norm(nn)
                Fp = np.stack([f1, f2, np.cross(f1, f2)], axis=1)             # columns: posed frame
                J[row, :, c0:c0 + 3] = np.eye(3)
                J[row, :, c0 + 3:c0 + per0] = sum(loc[i, :, 3 * t:3 * t + 3].dot(dv_pose[i, t]) for t in range(3))[:, pose_ids]
                J[row, :, off_ml + 3 * i:off_ml + 3 * i + 3] = Fp.dot(Fcan[i])
                J[row, :, c0 + per0:c0 + per] = sum(loc[i, :, 3 * t:3 * t + 3].dot(dv_beta[i, t]) for t in range(3))
            block('data', ((self.obs[f] - sim[ids]) * wts['data']).reshape(-1), -J.reshape(-1, n) * wts['data'])
        # ---- the jaw and the expressions of every frame
        if detailed:
            col = {pid: c for c, pid in enumerate(pose_ids)}
            for name, w in (('poseF', wts['poseF']), ('expr', wts['expr'])):
                for f in range(F):
                    c0 = off_fr + f * per
                    cols = [c0 + 3 + col[p] for p in self.face_ids] if name == 'poseF' else list(range(c0 + per0, c0 + per))
                    r = (self.pose[f, self.face_ids] if name == 'poseF' else self.expr[f]) * w
                    J = None
                    if want_jac:
                        J = np.zeros((r.size, n))
                        J[np.arange(r.size), cols] = w
                    block(name, r, J)
        r = np.concatenate(rs)
        return (r, np.vstack(Js)) if want_jac else r

    def run(self):
        cfg = self.cfg
        self.rigid_adjust()
        ann = list(cfg.opt_settings.weights['stagei_wt_annealing'])
        errs = {}
        for tidx, a in enumerate(ann):
            detailed = tidx > len(ann) - 3                                                      # chmosh.py:311
            wts = self.weights_for(a)
            pose_ids = self.pose_ids_for(detailed)

            def obj(x, want_jac):
                return self.face_residual(x, want_jac, pose_ids, wts, detailed)

            x, st = minimize_dogleg(obj, self.get_face_x(pose_ids, detailed), e_3=float(cfg.opt_settings.stagei_lr),
                                    delta_0=0.5, maxiter=int(cfg.opt_settings.maxiter))
            self.set_face_x(x, pose_ids, detailed)
            self.stats['r_evals'] += st.r_evals
            self.stats['j_evals'] += st.j_evals
            self.stats['iterations'] += st.iterations
            self.stats['minimizations'] += 1
            errs = {}
            self.face_residual(x, False, pose_ids, wts, detailed, per_term=errs)
        return errs


def face_oracle_stagei(stagei_frames, cfg, betas_fname, marker_meta):
    """The return dictionary of oracle.stagei.mosh_stagei, with the expressions as ``opt_models_expression``."""
    s = FaceOracle(stagei_frames, cfg, marker_meta, np.load(betas_fname)['betas'])
    errs = s.run()
    _, closest = NearestNeighbors(algorithm='kd_tree', n_neighbors=1).fit(s.can_v()).kneighbors(s.ml)
    sims_all = s.markers_sim_all()
    dbg = {'opt_models_trans': [t.copy() for t in s.trans], 'opt_models_pose': [p.copy() for p in s.pose],
           'opt_models_expression': [e.copy() for e in s.expr], 'stagei_errs': errs, 'stagei_markers_sim_all': sims_all,
           'stagei_markers_sim': [sims_all[f][s.lm_ids[f]] for f in range(s.n_frames)], 'stagei_markers_obs': s.obs,
           'stagei_labels_obs': s.labels_obs, 'oracle_stats': dict(s.stats)}
    return {'betas': s.betas.copy(), 'markers_latent': s.ml.copy(), 'latent_labels': s.latent_labels, 'marker_meta': marker_meta,
            'markers_latent_vids': {l: int(c[0]) for l, c in zip(s.latent_labels, closest.tolist())}, 'stagei_debug_details': dbg}


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
    s = FaceOracle(frames, cfg, case['marker_meta'], case['betas'])
    assert len(s.expr_ids) == 8
    s.rigid_adjust()
    wts = s.weights_for(0.25)
    pose_ids = s.pose_ids_for(True)
    assert {66, 67, 68} <= set(pose_ids.tolist())
    off_ml, off_fr, _, per, n = s.face_layout(pose_ids, True)
    npi, M = len(pose_ids), s.n_markers
    rng = np.random.default_rng(0)
    x0 = s.get_face_x(pose_ids, True)
    ids = np.arange(len(x0))
    frame_part = ids >= off_fr
    is_expr = frame_part & ((ids - off_fr) % per >= 3 + npi)
    x0 = x0 + rng.normal(0, 0.02, x0.shape) * (frame_part & ~is_expr) + rng.normal(0, 0.5, x0.shape) * is_expr
    r, J = s.face_residual(x0, True, pose_ids, wts, True)
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
        return s.face_residual(x, False, pose_ids, wts, True)
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
    ref = face_oracle_stagei(frames, cfg, fn, meta)
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
    ref = face_oracle_stagei(frames, cfg, fn, case['marker_meta'])
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
