"""The SMAL dog (``animal_dog``; reference: models/bodymodel_loader.py:126-131, chmosh.py:304-309,574-579,
prior/dog_body_prior.py:53-87): an LBS body with an 8-component max-mixture pose prior over 93 pose ids with gaps, the first
model whose prior sees a scattered set of pose ids (mosh2_model_desc.prior_ids).

CPU: the prior constants against the reference's formula, the pose partitions against the reference's id lists, the packs of
the other families unchanged, and the device source (single-thread host build) against the float64 oracle in Stage II and
Stage I.  ``-m gpu``: the CUDA library against the same oracle, the normal equations of a dog frame in both workspace layouts,
the workspace at the reference's marker counts, and launches that mix the dog with other models."""
import copy
import ctypes as C
import dataclasses
import pickle
from unittest import mock

import numpy as np
import pytest

from conftest import EmuStageIBackend, dense_obs, gpu_solve, run_oracle, stagei_case
from moshpp_b200 import chmosh, lib, synth
from moshpp_b200 import pack as _pack
from moshpp_b200 import stagei as product
from oracle import stagei as oracle_stagei
from oracle.prior import dog_oracle_prior

DOG = dict(frames=10, n_verts=1500)
DOG_JOINTS = [1, 3, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 30, 31, 32, 33, 34]


def _dog(cases, **kw):
    return cases('CD', **dict(DOG, **kw))


def _write_prior(path, d):
    with open(path, 'wb') as f:
        pickle.dump(d, f, protocol=pickle.HIGHEST_PROTOCOL)
    return str(path)


def _direct_neglogw(covs, weights):
    """-log of the reference's normalised weights, prior/dog_body_prior.py:77-83 as written (direct determinants)."""
    D = covs.shape[1]
    sqrdets = np.array([np.sqrt(np.linalg.det(c)) for c in covs])
    return -np.log(weights / ((2 * np.pi) ** (D / 2.) * (sqrdets / sqrdets.min())))



# ---- the prior constants ------------------------------------------------------------------------------------------------

def test_prior_constants_equal_the_reference_formula(tmp_path):
    d = synth.make_dog_prior()
    fn = _write_prior(tmp_path / 'dog.pkl', d)
    pr = _pack.create_dog_body_prior(fn)
    ids = np.arange(105).reshape(-1, 3)[DOG_JOINTS].reshape(-1)
    assert np.array_equal(_pack.DOG_BODY_IDS, ids) and len(ids) == 93
    covs = d['gmm_covs'][:, :, ids][:, ids]
    assert pr.means.shape == (8, 93) and pr.Q.shape == (8, 93, 93)
    assert np.array_equal(pr.means, d['gmm_means'][:, ids])
    assert np.abs(pr.neglogw - _direct_neglogw(covs, d['gmm_weights'])).max() < 1e-12
    ref = dog_oracle_prior(fn)             # the residual sqrt(.5) (x - mu) chol(inv S): its square is x^T Q x
    for k in range(8):
        q = 0.5 * ref.precs[k] @ ref.precs[k].T
        assert np.abs(pr.Q[k] - q).max() < 1e-12 * np.abs(q).max()
    assert np.abs(pr.neglogw + np.log(ref.weights)).max() < 1e-12
    # the weights spread over two orders of magnitude, the normalised constants lie close together
    assert d['gmm_weights'].max() / d['gmm_weights'].min() > 100 and np.ptp(pr.neglogw) < 1.0


def test_prior_constants_stay_finite_where_the_determinant_underflows(tmp_path):
    """Per-axis variances near 1e-4: det S = 0 in float64 at D = 93, and the reference's direct formula gives 0 / 0.  The log
    domain keeps the constants finite and equal to the direct formula on the same prior rescaled (the constants depend on the
    ratios of the determinants only)."""
    d = synth.make_dog_prior()
    small = dict(d, gmm_covs=d['gmm_covs'] * 1e-3)
    pr = _pack.create_dog_body_prior(_write_prior(tmp_path / 'small.pkl', small))
    ids = _pack.DOG_BODY_IDS
    covs = small['gmm_covs'][:, :, ids][:, ids]
    assert np.all([np.linalg.det(c) == 0.0 for c in covs])
    with np.errstate(divide='ignore', invalid='ignore'):
        assert not np.isfinite(_direct_neglogw(covs, d['gmm_weights'])).any()
    assert np.isfinite(pr.neglogw).all() and np.isfinite(pr.Q).all()
    want = _direct_neglogw(covs * 1e3, d['gmm_weights'])
    assert np.abs(pr.neglogw - want).max() < 1e-9
    with pytest.raises(ValueError):          # the oracle keeps the reference's direct formula and refuses such a prior
        dog_oracle_prior(str(tmp_path / 'small.pkl'))


def test_covariance_that_is_not_positive_definite_is_refused(tmp_path):
    d = synth.make_dog_prior()
    covs = d['gmm_covs'].copy()
    w, v = np.linalg.eigh(covs[3])
    w[10] = -w[10]
    covs[3] = (v * w) @ v.T
    with pytest.raises(ValueError, match='component 3'):
        _pack.create_dog_body_prior(_write_prior(tmp_path / 'bad.pkl', dict(d, gmm_covs=covs)))


# ---- pose partitions and packs ------------------------------------------------------------------------------------------

@pytest.mark.parametrize('toes', [False, True])
def test_pose_partitions_equal_the_reference_lists(toes):
    all_ids = list(range(105))
    body = [all_ids[i] for i in np.arange(0, 105).reshape([-1, 3])[DOG_JOINTS].reshape(-1)]     # chmosh.py:574-579
    ids = all_ids[:3] + body
    if not toes:
        ids = list(set(ids).difference(set(all_ids[30:36])))                                     # chmosh.py:645-647
    parts = _pack.pose_partitions('animal_dog', 105, optimize_fingers=True, optimize_face=True, optimize_toes=toes)
    assert parts['root'] == [0, 1, 2] and parts['body'] == body
    assert parts['finger'] == [] and parts['face'] == []
    assert parts['step1'] == sorted(ids) and parts['step2'] == sorted(ids)
    assert len(parts['step1']) == (96 if toes else 90)


def test_model_with_fewer_than_35_joints_is_refused():
    with pytest.raises(ValueError, match='34 joints'):
        _pack.pose_partitions('animal_dog', 3 * 34, False, False, False)


def test_dog_pack_carries_the_scattered_prior_ids(cases):
    case = _dog(cases)
    pk = case['pack']
    assert pk.model_type == 'animal_dog' and pk.n_joints == 35 and pk.p_red == 105
    assert pk.prior_k == 8 and pk.prior_d == 93 and np.array_equal(pk.prior_ids, _pack.DOG_BODY_IDS)
    assert len(pk.jangles_ids) == 0 and pk.finger_hi == pk.finger_lo and pk.n_dmpl == 0
    assert not set(range(30, 36)) & set(pk.free_step1 - 3) and len(pk.free_step1) == 3 + 90
    h = lib.DescHolder(pk)
    assert h.desc.prior_ids and [h.desc.prior_ids[i] for i in range(93)] == list(_pack.DOG_BODY_IDS)


@pytest.mark.parametrize('name', ['C1', 'C2', 'C3', 'C4', 'CF', 'CH'])
def test_packs_of_the_other_families_are_unchanged(cases, name):
    """A contiguous prior keeps prior_off and no id table; its constants are those of the family's own prior."""
    case = cases(name)
    pk = case['pack']
    assert len(pk.prior_ids) == 0 and not lib.DescHolder(pk).desc.prior_ids
    cfg = case['cfg']
    if pk.model_type == 'mano':
        assert pk.prior_k == 0
        return
    fn = cfg.moshpp.pose_body_prior_fname
    pr = (_pack.create_horse_body_prior(fn) if pk.model_type == 'animal_horse'
          else _pack.create_gmm_body_prior(fn, exclude_hands=pk.model_type in ('smplh', 'smplx')))
    assert pk.prior_off == 3 and pk.prior_d == {'smpl': 69, 'animal_horse': 81}.get(pk.model_type, 63)
    for a, b in ((pk.prior_means, pr.means), (pk.prior_Q, pr.Q), (pk.prior_neglogw, pr.neglogw)):
        assert a.dtype == b.dtype and a.tobytes() == b.tobytes()


def test_stageii_without_a_prior_file_raises_key_error(cases):
    case = _dog(cases)
    cfg = copy.deepcopy(case['cfg'])
    cfg.moshpp.pose_body_prior_fname = None
    with pytest.raises(KeyError, match='pose'):
        chmosh.prepare_stageii(cfg, case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])


def test_motion_keeps_the_joints_outside_the_prior_at_rest(cases):
    pose = _dog(cases)['gt_pose']
    rest = sorted(set(range(3, 105)) - set(_pack.DOG_BODY_IDS)) + list(range(30, 36))
    assert np.abs(pose[:, rest]).max() == 0 and np.abs(pose[:, _pack.DOG_BODY_IDS]).max() > 0.05



def test_prepare_cfg_needs_the_weights_for_the_dog(tmp_path):
    """The yaml has no opt_weights block for the animal models: the weights come from opt_settings.weights."""
    import json
    import os
    from moshpp_b200.cfg import STAGEII_WEIGHTS, prepare_cfg
    fn = os.path.join(str(tmp_path), 'mocap', 'DS', 'dog01', 'trot.npz')
    os.makedirs(os.path.dirname(fn))
    np.savez(fn, markers=np.ones((3, 2, 3)), labels=np.array(['A', 'B']), frame_rate=100.0)
    with open(os.path.join(os.path.dirname(fn), 'settings.json'), 'w') as f:
        json.dump({'gender': 'male'}, f)
    kw = {'mocap.fname': fn, 'dirs.work_base_dir': str(tmp_path / 'w'), 'dirs.support_base_dir': str(tmp_path / 's'),
          'surface_model.type': 'animal_dog'}
    with pytest.raises(KeyError, match='opt_settings.weights'):
        prepare_cfg(**kw).opt_settings.weights
    cfg = prepare_cfg(**dict(kw, **{'opt_settings.weights': dict(STAGEII_WEIGHTS)}))
    assert cfg.surface_model.type == 'animal_dog' and cfg.opt_settings.weights['stageii_wt_poseB'] == STAGEII_WEIGHTS['stageii_wt_poseB']

# ---- Stage II on the device source ---------------------------------------------------------------------------------------

def _check_f64(case, res, out, tol_pose, tol_trans, rtol, atol):
    dbg = out['stageii_debug_details']
    fid = dbg['frame_ids']
    assert np.array_equal(np.nonzero(res.status & lib.ST_SOLVED)[0], fid)
    assert np.abs(res.pose[fid] - out['_pose_reduced']).max() < tol_pose
    assert np.abs(res.fullpose[fid] - out['fullpose']).max() < tol_pose
    assert np.abs(res.trans[fid] - out['trans']).max() < tol_trans
    assert res.counters[fid, 2].sum() == dbg['oracle_stats']['j_evals']
    assert np.allclose(res.errs[fid, 0], dbg['stageii_errs']['data'], rtol=rtol, atol=atol)
    assert np.allclose(res.errs[fid, 1], dbg['stageii_errs']['poseB'], rtol=rtol, atol=atol)
    assert np.all(res.errs[fid, 3] == 0)                    # no joint-angle term
    rest = sorted(set(range(3, 105)) - set(_pack.DOG_BODY_IDS)) + list(range(30, 36))
    assert np.abs(res.pose[fid][:, rest]).max() == 0


def test_f64_device_source_equals_oracle(cases, emu):
    case = _dog(cases)
    out = run_oracle(case)
    res = emu(case, precision=lib.MOSH2_F64)
    _check_f64(case, res, out, 1e-9, 1e-10, 1e-8, 1e-12)
    assert res.counters[out['stageii_debug_details']['frame_ids'], 3].sum() == out['stageii_debug_details']['oracle_stats']['minimizations']


def test_solve_moves_between_mixture_components(cases):
    """The fixture exercises the max-mixture selection: the component of the solved poses changes within the case."""
    case = _dog(cases)
    out = run_oracle(case)
    pr = dog_oracle_prior(case['cfg'].moshpp.pose_body_prior_fname)
    comp = [pr.select(x)[0] for x in out['_pose_reduced'][:, _pack.DOG_BODY_IDS]]
    assert len(set(comp)) > 1, comp


def test_stageii_output_reports_poseB_only(cases, emu):
    case = _dog(cases)
    pk, opts, flags = chmosh.prepare_stageii(case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'],
                                             case['marker_meta'])
    assert np.array_equal(pk.prior_ids, case['pack'].prior_ids) and pk.prior_Q.tobytes() == case['pack'].prior_Q.tobytes()
    assert chmosh.default_schedule(pk.model_type, 'fast', pk.n_dmpl) == chmosh.default_schedule('animal_horse', 'fast', 0)
    obs, vis = dense_obs(case)
    res = emu(case)
    data = chmosh.assemble_stageii_data(res, obs, vis, case['latent_labels'], pk, flags, False)
    assert set(data['stageii_debug_details']['stageii_errs']) == {'data', 'poseB', 'velo'}


def _permuted(pk, seed=3):
    """The same prior with its dimensions in another order: pose ids, means and Q permuted together."""
    p = np.random.default_rng(seed).permutation(pk.prior_d)
    return dataclasses.replace(pk, prior_ids=np.ascontiguousarray(pk.prior_ids[p]), prior_means=np.ascontiguousarray(pk.prior_means[:, p]),
                               prior_Q=np.ascontiguousarray(pk.prior_Q[:, p][:, :, p]))


def test_prior_ids_are_read_per_model_in_a_multi_model_job(cases):
    """Two dog subjects in one multi-model job, the second with its prior dimensions in another order (the same prior): each
    sequence equals its subject's own batch job bit for bit, and the permuted subject equals the unpermuted one to rounding.
    A kernel that read the first model's id table for both would hold the second dog to a scrambled prior."""
    from moshpp_b200 import build
    handle = C.CDLL(build.build_emu())
    a, b = _dog(cases), _dog(cases, seq_idx=1)
    pa, pb = a['pack'], _permuted(b['pack'])
    assert chmosh.kernel_shape_key(pa) == chmosh.kernel_shape_key(pb) and not np.array_equal(pa.prior_ids, pb.prior_ids)
    ova, ovb = dense_obs(a), dense_obs(b)
    opt = lib.make_options(a['cfg'].opt_settings.weights)
    sched = lib.make_schedule(4, 3, 2, 0)
    holders = [lib.DescHolder(pa), lib.DescHolder(pb)]
    descs = (C.POINTER(lib.ModelDesc) * 2)(*[C.pointer(h.desc) for h in holders])
    counts = np.array([10, 10], dtype=np.int32)
    mos = np.array([0, 1], dtype=np.int32)
    obs = np.ascontiguousarray(np.concatenate([ova[0], ovb[0]]), dtype=np.float64)
    vis = np.ascontiguousarray(np.concatenate([ova[1], ovb[1]]), dtype=np.uint8)
    multi = lib.ResultArrays(20, lib.pack_dims(pa))
    assert handle.mosh2_emu_solve_multi(descs, 2, C.byref(opt), 2, lib._ptr(counts, lib._i32p), lib._ptr(mos, lib._i32p),
                                        lib._ptr(obs, lib._f64p), lib._ptr(vis, lib._u8p), C.byref(sched), lib.MOSH2_F64,
                                        C.byref(multi.c)) == 0

    def alone(pk, ov):
        res = lib.ResultArrays(10, lib.pack_dims(pk))
        o, v = np.ascontiguousarray(ov[0], dtype=np.float64), np.ascontiguousarray(ov[1], dtype=np.uint8)
        one = np.array([10], dtype=np.int32)
        assert handle.mosh2_emu_solve_batch(C.byref(lib.DescHolder(pk).desc), C.byref(opt), 1, lib._ptr(one, lib._i32p),
                                            lib._ptr(o, lib._f64p), lib._ptr(v, lib._u8p), C.byref(sched), lib.MOSH2_F64,
                                            C.byref(res.c)) == 0
        return res
    ra, rb, rb0 = alone(pa, ova), alone(pb, ovb), alone(b['pack'], ovb)
    for name in ('pose', 'trans', 'errs', 'status'):
        assert np.array_equal(getattr(multi, name)[:10], getattr(ra, name)), name
        assert np.array_equal(getattr(multi, name)[10:], getattr(rb, name)), name
    assert np.abs(rb.pose - rb0.pose).max() < 1e-9 and np.array_equal(rb.counters, rb0.counters)


# ---- Stage I -----------------------------------------------------------------------------------------------------------

def _stagei(cases, backend, tol):
    case, cfg, frames = stagei_case(cases, 'CD', 4, **DOG)
    cfg.opt_settings.maxiter = 3
    ref = oracle_stagei.mosh_stagei(frames, cfg, marker_meta=case['marker_meta'])
    out = product.mosh_stagei(frames, cfg, marker_meta=case['marker_meta'], backend=backend)
    assert np.abs(out['betas'] - ref['betas']).max() < tol
    assert np.abs(out['markers_latent'] - ref['markers_latent']).max() < tol
    do, dr = out['stagei_debug_details'], ref['stagei_debug_details']
    for a, b in zip(do['opt_models_pose'], dr['opt_models_pose']):
        assert np.abs(a - b).max() < tol
    for a, b in zip(do['opt_models_trans'], dr['opt_models_trans']):
        assert np.abs(a - b).max() < tol
    assert set(do['stagei_errs']) == set(dr['stagei_errs']) and 'poseB' in dr['stagei_errs'] and 'poseB_jangles' not in dr['stagei_errs']
    for k, v in dr['stagei_errs'].items():
        assert abs(do['stagei_errs'][k] - v) <= 1e-5 * abs(v) + 100 * tol, k
    st, rs = do['b200'], dr['oracle_stats']
    assert st['linearisations'] == rs['j_evals'] and st['iterations'] == rs['iterations'] and st['minimisations'] == 4
    assert np.abs(out['betas'][:cfg.surface_model.num_betas]).max() > 1e-3


def test_stagei_on_the_device_source_equals_oracle(cases):
    _stagei(cases, EmuStageIBackend(), 1e-9)


# ---- normal equations of a dog frame ------------------------------------------------------------------------------------

# float32: the CPU twin's maxima over Step 1 and Step 2; the bounds are 4x these (as in tests/test_gpu_normal_equations.py)
DOG_F32 = dict(J=6.0e-6, r=4.1e-7, vp=3.3e-7, markers=4.1e-7, A=4.1e-6, g=1.0e-5, sse=3.6e-7, data=1.1e-8)


def _ne():
    import test_gpu_normal_equations as ne
    return ne


def _errors(case, pk, opts, step, obs, vis, x, out, precision, tc=False):
    ne = _ne()
    with mock.patch.dict(ne.TWIN_F32, {'CD': DOG_F32}):
        return ne.normal_equation_errors(case, 'CD', pk, opts, step, obs, vis, x, out, precision, tc=tc)


@pytest.fixture(scope='module')
def emu_lin():
    from moshpp_b200 import build
    handle = C.CDLL(build.build_emu())

    def run(pk, opts, obs, vis, x, step, precision):
        F, M = obs.shape[0], pk.n_markers
        n = len(pk.free_step2 if step == 2 else pk.free_step1)
        h = lib.DescHolder(pk)
        out = dict(errs=np.zeros((F, len(lib.ERR_NAMES))), markers_sim=np.zeros((F, M, 3)), r=np.zeros((F, 3 * M)),
                   vp=np.zeros((F, 3 * M, 3)), A=np.zeros((F, n, n)), g=np.zeros((F, n)), J=np.zeros((F, 3 * M, n)))
        c = lib.LinOut(*[lib._ptr(out[k], lib._f64p) for k in ('errs', 'markers_sim', 'r', 'vp', 'A', 'g', 'J')])
        prec = {'f32': lib.MOSH2_F32, 'f64': lib.MOSH2_F64}[precision]
        assert handle.mosh2_emu_linearize_precision(C.byref(h.desc), C.byref(opts), F, lib._ptr(obs, lib._f64p), lib._ptr(vis, lib._u8p),
                                                    int(step), 1, lib._ptr(x, lib._f64p), prec, C.byref(c)) == 0
        return out
    return run


@pytest.mark.parametrize('precision', ['f64', 'f32'])
@pytest.mark.parametrize('step', [1, 2])
def test_device_source_normal_equations_equal_float64(cases, emu, emu_lin, step, precision):
    ne = _ne()
    case = _dog(cases)
    pk, opts = ne._prepare(case)
    obs, vis, x = ne.lin_inputs(case, emu(case))
    out = emu_lin(pk, opts, obs, vis, x, step, precision)
    st = _errors(case, pk, opts, step, obs, vis, x, out, precision)
    print('CD', step, precision, {k: float('%.2g' % v) for k, v in st.items()})


# ---- the workspace at the reference's marker counts ----------------------------------------------------------------------

def _relayout(case, n_markers):
    labels, vids, meta = synth.make_layout(case['model'], 'animal_dog', n_markers, 0)
    ml = synth.make_markers_latent(case['model'], 'animal_dog', case['betas'], 16, vids, meta)
    return labels, meta, ml


def _packs_at(cases, n_markers):
    case = _dog(cases)
    labels, meta, ml = _relayout(case, n_markers)
    pk2, _, _ = chmosh.prepare_stageii(case['cfg'], ml, labels, case['betas'], meta)
    cfg = copy.deepcopy(case['cfg'])
    cfg.moshpp.optimize_betas = True
    s = product.StageI([{l: np.zeros(3) for l in labels}], cfg, meta, backend=object())
    pk1 = s.pack_for(True)
    assert pk2.n_markers == pk1.n_markers == n_markers and pk1.n_dmpl == 16
    return case, pk2, pk1, labels, meta, ml


@pytest.mark.parametrize('n_markers', [65, 90])
def test_workspace_plan_fits(cases, n_markers):
    from moshpp_b200 import build
    fn = C.CDLL(build.build_emu()).mosh2_emu_plan
    fn.argtypes = [C.POINTER(lib.ModelDesc), C.c_int32, C.c_int32, C.POINTER(C.c_int64)]
    fn.restype = C.c_int32
    _, pk2, pk1, *_ = _packs_at(cases, n_markers)
    for pk in (pk2, pk1):
        for precision in (lib.MOSH2_F32, lib.MOSH2_F64):
            for multi in (0, 1):
                out = (C.c_int64 * 5)()
                assert fn(C.byref(lib.DescHolder(pk).desc), precision, multi, out) == 0
                assert out[0] <= out[4], (n_markers, pk.n_dmpl, precision, multi, list(out))


# ==== on the H100 ==========================================================================================================

@pytest.mark.gpu
def test_f64_kernel_equals_oracle(cases):
    case = _dog(cases)
    out = run_oracle(case)
    res = gpu_solve(case, precision='f64')
    _check_f64(case, res, out, 1e-8, 1e-9, 1e-7, 1e-10)
    mk = np.concatenate(out['stageii_debug_details']['markers_sim'])
    _, vis = dense_obs(case)
    fid = out['stageii_debug_details']['frame_ids']
    assert np.abs(res.markers_sim[fid][vis[fid]] - mk).max() < 1e-9


@pytest.mark.gpu
def test_f32_kernel_within_stated_tolerance(cases):
    """The float32 bounds of tests/test_gpu_parity.py for the horse (BASELINE.md section 4)."""
    case = _dog(cases)
    out = run_oracle(case)
    res = gpu_solve(case, precision='f32')
    dbg = out['stageii_debug_details']
    fid = dbg['frame_ids']
    dp = np.abs(res.pose[fid] - out['_pose_reduced'])
    assert dp[:, :66].max() < 1e-3 and dp.max() < 1e-2
    assert np.abs(res.trans[fid] - out['trans']).max() < 1e-4
    assert np.abs(res.errs[fid, 0] / dbg['stageii_errs']['data'] - 1).max() < 1e-2
    mk = np.concatenate(dbg['markers_sim'])
    _, vis = dense_obs(case)
    assert np.abs(res.markers_sim[fid][vis[fid]] - mk).max() < 1e-4


@pytest.mark.gpu
def test_drop_in_callable_with_the_dog_model(cases):
    case = _dog(cases)
    out = chmosh.mosh_stageii(mocap_fname=case['mocap_fname'], cfg=case['cfg'], markers_latent=case['markers_latent'],
                              latent_labels=case['latent_labels'], betas=case['betas'], marker_meta=case['marker_meta'],
                              precision='f64', chunk_len=0)
    ref = run_oracle(case)
    assert np.abs(out['fullpose'] - ref['fullpose']).max() < 1e-8 and np.abs(out['trans'] - ref['trans']).max() < 1e-9
    e, r = out['stageii_debug_details']['stageii_errs'], ref['stageii_debug_details']['stageii_errs']
    assert set(e) == set(r) == {'data', 'poseB', 'velo'}
    for k in ('data', 'poseB'):
        assert np.allclose(e[k], r[k], rtol=1e-7, atol=1e-10)


@pytest.fixture(scope='module')
def dog_states():
    cache = {}

    def get(case):
        if 'x' not in cache:
            cache['x'] = _ne().lin_inputs(case, gpu_solve(case, precision='f64'))
        return cache['x']
    return get


@pytest.mark.gpu
@pytest.mark.parametrize('layout', ['shared', 'global'])
@pytest.mark.parametrize('precision', ['f64', 'f32'])
@pytest.mark.parametrize('step', [1, 2])
def test_kernel_normal_equations_equal_float64(cases, dog_states, step, precision, layout, monkeypatch):
    """The normal equations of dog frames at given states, in the shared-memory layout and in the global-workspace layout
    (MOSH2_DEV_BIG: A, its factor and the Jacobian tiles in a per-CTA global workspace)."""
    ne = _ne()
    case = _dog(cases)
    pk, opts = ne._prepare(case)
    obs, vis, x = dog_states(case)
    if layout == 'global':
        monkeypatch.setenv('MOSH2_DEV_BIG', '1')
    out = ne.gpu_linearize(pk, opts, obs, vis, x, step, precision)
    monkeypatch.delenv('MOSH2_DEV_BIG', raising=False)
    st = _errors(case, pk, opts, step, obs, vis, x, out, precision, tc=precision == 'f32' and layout == 'shared')
    print('CD', step, precision, layout, {k: float('%.2g' % v) for k, v in st.items()})


@pytest.mark.gpu
@pytest.mark.parametrize('precision', ['f64', 'f32'])
def test_kernel_solve_in_the_global_workspace_layout_equals_oracle(cases, precision, monkeypatch):
    case = _dog(cases)
    out = run_oracle(case)
    monkeypatch.setenv('MOSH2_DEV_BIG', '1')
    res = gpu_solve(case, precision=precision)
    monkeypatch.delenv('MOSH2_DEV_BIG')
    fid = out['stageii_debug_details']['frame_ids']
    dp = np.abs(res.pose[fid] - out['_pose_reduced']).max()
    assert dp < (1e-8 if precision == 'f64' else 1e-3), dp


@pytest.mark.gpu
def test_stagei_on_the_gpu_equals_oracle(cases):
    _stagei(cases, None, 1e-6)


@pytest.mark.gpu
@pytest.mark.parametrize('n_markers', [65, 90])
def test_kernel_runs_at_the_reference_marker_counts(cases, n_markers):
    """65 and 90 markers: the Stage-II model solves frames in both precisions, and Stage I linearises its picked frames."""
    case, pk2, pk1, labels, meta, ml = _packs_at(cases, n_markers)
    gt = synth.forward_markers(pk2, case['gt_pose'][:4], case['gt_trans'][:4])
    vis = np.ones(gt.shape[:2], dtype=bool)
    opts = lib.make_options(case['cfg'].opt_settings.weights)
    sols = {}
    for name, prec in (('f32', lib.MOSH2_F32), ('f64', lib.MOSH2_F64)):
        model = lib.Model(pk2, device=0)
        try:
            res = model.solve(gt, vis, opts, chunk_len=0, chunk_warmup=0, precision=prec)
        finally:
            model.close()
        assert (res.status & lib.ST_SOLVED).all() and np.isfinite(res.pose).all()
        sols[name] = res
    assert np.abs(sols['f32'].pose - sols['f64'].pose)[:, :3].max() < 1e-2
    # the Stage-I pack (the shape as a linear block of 16 coefficients) linearised at the solved states
    x = np.zeros((4, pk1.nx))
    x[:, :3], x[:, 3:3 + pk1.p_red] = sols['f64'].trans, sols['f64'].pose
    obs, v8 = np.ascontiguousarray(gt), np.ascontiguousarray(vis, dtype=np.uint8)
    for precision in ('f32', 'f64'):
        out = _ne().gpu_linearize(pk1, opts, obs, v8, np.ascontiguousarray(x), 2, precision)
        assert out['A'].shape == (4, len(pk1.free_step2), len(pk1.free_step2)) and np.isfinite(out['A']).all()
        assert np.all(out['errs'][:, 1] > 0)


@pytest.mark.gpu
def test_subjects_call_with_a_dog_and_two_smplh_subjects(tmp_path):
    """mosh_stageii_subjects with one dog and two SMPL-H subjects: two launches (the dog has a kernel shape of its own), and
    every capture equals the single-subject call of its subject."""
    root = str(tmp_path)
    subs = []
    for k, (config, fr) in enumerate((('C2', (10, 8)), ('CD', (10,)), ('C2', (9,)))):
        case, fnames = synth.make_subject(root, config, fr, n_verts=1500, seq_idx=k)
        subs.append(dict(cfg=case['cfg'], mocap_fnames=fnames, markers_latent=case['markers_latent'],
                         latent_labels=case['latent_labels'], betas=case['betas'], marker_meta=case['marker_meta']))
    kw = dict(precision='f64', chunk_len=0)
    outs = chmosh.mosh_stageii_subjects(subs, **kw)
    assert [len(o) for o in outs] == [2, 1, 1]
    batch = outs[1][0]['stageii_debug_details']['b200']['batch']
    assert batch['launches'] == 2
    for s, so in zip(subs, outs):
        alone = chmosh.mosh_stageii_subjects([s], **kw)[0]
        for a, b in zip(so, alone):
            assert np.array_equal(a['fullpose'], b['fullpose']) and np.array_equal(a['trans'], b['trans'])
            for k, v in b['stageii_debug_details']['stageii_errs'].items():
                assert np.array_equal(a['stageii_debug_details']['stageii_errs'][k], v), k
    assert set(outs[1][0]['stageii_debug_details']['stageii_errs']) == {'data', 'poseB', 'velo'}


@pytest.mark.gpu
@pytest.mark.parametrize('precision', ['f32', 'f64'])
def test_kernel_reads_the_prior_ids_of_each_model_in_a_multi_model_launch(cases, precision):
    """The GPU twin of test_prior_ids_are_read_per_model_in_a_multi_model_job, chunked: one multi-model launch of a dog and a
    dog whose prior dimensions are permuted equals a batch job of each, bit for bit."""
    a, b = _dog(cases), _dog(cases, seq_idx=1)
    pa, pb = a['pack'], _permuted(b['pack'])
    prec = {'f32': lib.MOSH2_F32, 'f64': lib.MOSH2_F64}[precision]
    sched = dict(chunk_len=4, chunk_warmup=3, warmup_full=2, first_extra=0, precision=prec)
    opts = lib.make_options(a['cfg'].opt_settings.weights)
    ova, ovb = dense_obs(a), dense_obs(b)
    models = [lib.Model(pa, device=0), lib.Model(pb, device=0)]
    try:
        job = lib.multi_job(models, [0, 1], [10, 10], opts, **sched)
        job.upload(np.concatenate([ova[0], ovb[0]]), np.concatenate([ova[1], ovb[1]]))
        job.launch()
        job.sync()
        multi = job.download()
        job.close()
        for k, (m, ov) in enumerate(zip(models, (ova, ovb))):
            one = m.job([10], opts, **sched)
            one.upload(*ov)
            one.launch()
            one.sync()
            r = one.download()
            one.close()
            for name in ('pose', 'trans', 'errs', 'status'):
                assert np.array_equal(getattr(multi, name)[10 * k:10 * (k + 1)], getattr(r, name)), (k, name)
    finally:
        for m in models:
            m.close()
