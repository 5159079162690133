"""Parity tests proper: the CUDA library (through the C-ABI) against the float64 oracle on an H100."""
import numpy as np
import pytest

from conftest import dense_obs, gpu_solve, run_oracle
from moshpp_b200 import lib

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('name', ['C1', 'C2', 'C3', 'C4', 'CF', 'CH'])
def test_f64_kernel_equals_oracle(cases, name):
    case = cases(name)
    out = run_oracle(case)
    res = gpu_solve(case, precision='f64')
    dbg = out['stageii_debug_details']
    fid = dbg['frame_ids']
    assert np.array_equal(np.nonzero(res.status & lib.ST_SOLVED)[0], fid)
    assert np.abs(res.pose[fid] - out['_pose_reduced']).max() < 1e-8
    assert np.abs(res.fullpose[fid] - out['fullpose']).max() < 1e-8
    assert np.abs(res.trans[fid] - out['trans']).max() < 1e-9
    if 'dmpls' in out:
        assert np.abs(res.dmpls[fid, :out['dmpls'].shape[1]] - out['dmpls']).max() < 1e-8
    if 'expression' in out:
        pk = case['pack']
        assert np.abs(res.dmpls[fid, pk.n_dmpl - pk.n_expr:pk.n_dmpl] - out['expression'][:, :pk.n_expr]).max() < 1e-8
    assert res.counters[fid, 2].sum() == dbg['oracle_stats']['j_evals']
    for k, col in zip(lib.ERR_NAMES, range(len(lib.ERR_NAMES))):
        if k in dbg['stageii_errs'] and k not in ('velo', 'extrap_dmpl'):
            assert np.allclose(res.errs[fid, col], dbg['stageii_errs'][k], rtol=1e-7, atol=1e-10)
    mk = np.concatenate(dbg['markers_sim'])
    _, vis = dense_obs(case)
    assert np.abs(res.markers_sim[fid][vis[fid]] - mk).max() < 1e-9


@pytest.mark.parametrize('name', ['C1', 'C2', 'C3', 'C4', 'CF', 'CH'])
def test_f32_kernel_within_stated_tolerance(cases, name):
    """Tolerances of BASELINE.md section 4 for the fp32 path (sequential mode)."""
    case = cases(name)
    out = run_oracle(case)
    res = gpu_solve(case, precision='f32')
    dbg = out['stageii_debug_details']
    fid = dbg['frame_ids']
    bd = min(case['pack'].body_dof, 66)
    dp = np.abs(res.pose[fid] - out['_pose_reduced'])
    assert dp[:, :bd].max() < (5e-3 if name == "C4" else 1e-3)   # rad, root + body (C4: hand-only model, wrist weakly observed)
    assert dp.max() < 1e-2                              # weakly observed finger PCA coefficients
    assert np.abs(res.trans[fid] - out['trans']).max() < 1e-4   # m
    sse = dbg['stageii_errs']['data']
    assert np.abs(res.errs[fid, 0] / sse - 1).max() < 1e-2     # final marker residual within 1 %
    mk = np.concatenate(dbg['markers_sim'])
    _, vis = dense_obs(case)
    # (CF: the expression coefficients are nearly flat directions of the objective -- 0.15 mm measured on one face marker with
    # pose, translation and residual inside their tolerances; such models run float64 by default, chmosh.default_schedule)
    assert np.abs(res.markers_sim[fid][vis[fid]] - mk).max() < (3e-4 if name == 'CF' else 1e-4)


def test_chunked_kernel_equals_oracle_chunked(cases):
    case = cases('C2')
    out = run_oracle(case, chunk=(5, 2))
    res = gpu_solve(case, chunk_len=5, warmup=2, precision='f64')
    fid = out['stageii_debug_details']['frame_ids']
    assert np.abs(res.pose[fid] - out['_pose_reduced']).max() < 1e-8


def test_chunk_warmup_converges_on_gpu(cases):
    case = cases('C2', frames=160)
    seq = gpu_solve(case, precision='f64')
    ok = (seq.status & lib.ST_SOLVED) != 0
    e = [np.abs(gpu_solve(case, chunk_len=32, warmup=W, precision='f64').pose - seq.pose)[ok].max() for W in (0, 48, 96)]
    assert e[1] < 1e-3 and e[2] < 1e-6, e


def test_skipped_frames_and_flags(cases):
    case = cases('C1')
    obs, vis = dense_obs(case)
    vis = vis.copy()
    vis[3] = False
    res = gpu_solve(case, obs_vis=(obs, vis))
    assert res.status[3] == lib.ST_SKIPPED
    assert not (res.status[1] & lib.ST_HAS_VELO) and (res.status[2] & lib.ST_HAS_VELO)
    assert np.all(res.fullpose[3] == 0)


def test_full_size_c2_properties(cases):
    """BASELINE config 2 at full size (V=6890, 500 frames): size-independent properties."""
    case = cases('C2', frames=500, n_verts=None)
    obs, vis = dense_obs(case)
    res = gpu_solve(case, chunk_len=4, warmup=64, precision='f32')
    ok = (res.status & lib.ST_SOLVED) != 0
    assert ok.sum() == (vis.any(1)).sum()
    # solved markers reproduce the observations to about the 1 mm noise floor
    d = np.linalg.norm(res.markers_sim - obs, axis=-1)[vis]
    assert np.sqrt((d ** 2).mean()) < 2.5e-3
    # fullpose is the PCA expansion of the reduced pose (smpl_fast_derivatives.py:194-204)
    pk = case['pack']
    full = np.concatenate([res.pose[:, :pk.body_dof], pk.hands_mean[None] + res.pose[:, pk.body_dof:] @ pk.hand_comps], 1)
    assert np.abs(full[ok] - res.fullpose[ok]).max() < 1e-5
    # toes are frozen (chmosh.py:646-647)
    assert np.abs(res.pose[ok][:, 30:36]).max() == 0
    # chunked == sequential within the warm-up bound
    seq = gpu_solve(case, precision='f32')
    assert np.abs(seq.pose - res.pose)[ok][:, :66].max() < 2e-3


def test_drop_in_callable_matches_reference_layout(cases):
    """Called exactly like MoSh.mosh_stageii calls its plug-in (mosh_head.py:280-286); the return dict has
    the keys / shapes / list lengths of chmosh.py:726-741."""
    from moshpp_b200.chmosh import mosh_stageii
    case = cases('C3')
    out = mosh_stageii(mocap_fname=case['mocap_fname'], cfg=case['cfg'], markers_latent=case['markers_latent'],
                       latent_labels=case['latent_labels'], betas=case['betas'], marker_meta=case['marker_meta'],
                       v_template_fname=None)
    ref = run_oracle(case)
    assert set(out.keys()) >= {'fullpose', 'trans', 'dmpls', 'stageii_debug_details'}
    n = len(ref['fullpose'])
    assert out['fullpose'].shape == ref['fullpose'].shape and out['fullpose'].dtype == np.float64
    assert out['trans'].shape == (n, 3) and out['dmpls'].shape == ref['dmpls'].shape
    dbg, rdbg = out['stageii_debug_details'], ref['stageii_debug_details']
    for k in ('stageii_errs', 'markers_sim', 'markers_obs', 'labels_obs', 'markers_orig', 'labels_orig',
              'mocap_fname', 'mocap_frame_rate', 'mocap_time_length'):
        assert k in dbg
    assert set(dbg['stageii_errs'].keys()) == set(rdbg['stageii_errs'].keys())
    for k, v in rdbg['stageii_errs'].items():
        assert dbg['stageii_errs'][k].shape == v.shape
        assert np.allclose(dbg['stageii_errs'][k], v, rtol=2e-2, atol=1e-3)
    assert dbg['labels_obs'] == rdbg['labels_obs']
    assert all(a.shape == b.shape for a, b in zip(dbg['markers_sim'], rdbg['markers_sim']))
    assert np.abs(np.concatenate(dbg['markers_obs']) - np.concatenate(rdbg['markers_obs'])).max() == 0
    assert np.abs(out['trans'] - ref['trans']).max() < 1e-4


def test_drop_in_callable_with_face_expressions(cases):
    """optimize_face (SURVEY.md 8(f-4)): jaw + expression coefficients; return layout of chmosh.py:723-724,736 and the
    AMASS writer's `expression` key."""
    from moshpp_b200 import amass_io
    from moshpp_b200.chmosh import mosh_stageii
    case = cases('CF')
    out = mosh_stageii(mocap_fname=case['mocap_fname'], cfg=case['cfg'], markers_latent=case['markers_latent'],
                       latent_labels=case['latent_labels'], betas=case['betas'], marker_meta=case['marker_meta'],
                       precision='f64', chunk_len=0)
    ref = run_oracle(case)
    assert 'dmpls' not in out and out['expression'].shape == ref['expression'].shape
    assert np.abs(out['expression'] - ref['expression']).max() < 1e-8
    assert np.abs(out['fullpose'] - ref['fullpose']).max() < 1e-8
    dbg, rdbg = out['stageii_debug_details'], ref['stageii_debug_details']
    assert set(dbg['stageii_errs'].keys()) == set(rdbg['stageii_errs'].keys()) >= {'poseF', 'expr'}
    for k in ('poseF', 'expr'):
        assert np.allclose(dbg['stageii_errs'][k], rdbg['stageii_errs'][k], rtol=1e-7, atol=1e-10)
    assert np.abs(out['fullpose'][:, 66:69]).max() > 1e-3          # the jaw moved
    merged = amass_io.merge_stageii(out, dict(betas=case['betas'], markers_latent=case['markers_latent'],
                                              latent_labels=case['latent_labels']), case['cfg'], 0.0)
    npz = amass_io.load_as_amass_npz(merged)
    assert npz['expression'].shape == (len(out['fullpose']), case['cfg'].surface_model.num_expressions)
    assert npz['pose_jaw'].shape == (len(out['fullpose']), 3)


@pytest.mark.parametrize('name', ['C2', 'CF'])
def test_f32_global_workspace_layout_matches_shared_memory_layout(cases, name, monkeypatch):
    """Models whose normal equations do not fit the shared memory (e.g. SMPL-X with 80 expression coefficients) run
    with A, its factor and the Jacobian tiles in a per-block global workspace and J^T J on the CUDA cores; the same
    small case through both layouts must agree to f32 round-off and stay inside the f32 tolerances."""
    case = cases(name)
    a = gpu_solve(case, precision='f32')
    monkeypatch.setenv('MOSH2_DEV_BIG', '1')
    b = gpu_solve(case, precision='f32')
    monkeypatch.delenv('MOSH2_DEV_BIG')
    out = run_oracle(case)
    fid = out['stageii_debug_details']['frame_ids']
    bd = min(case['pack'].body_dof, 66)
    assert np.array_equal(a.status, b.status)
    assert np.abs(b.pose[fid] - out['_pose_reduced'])[:, :bd].max() < 1e-3
    assert np.abs(b.trans[fid] - out['trans']).max() < 1e-4
    # (each layout is inside the f32 tolerance of the oracle; against each other that allows twice the tolerance)
    assert np.abs(a.pose - b.pose)[:, :bd].max() < 2e-3 and np.abs(a.trans - b.trans).max() < 2e-4


def test_library_is_the_cuda_build():
    from moshpp_b200 import lib
    L = lib.load_library()
    assert L.mosh2_device_count() >= 1
    maps = open('/proc/self/maps').read()
    assert 'libmosh2.so' in maps


def test_tf32_jtj_building_block():
    """Stand-alone kernel (tests/tc): J^T J on the tensor cores with the split-TF32 / separate-accumulator scheme the
    Stage-II kernel uses (its own device function), against a float64 product, for the operand shapes of all model
    families."""
    import subprocess
    from moshpp_b200 import build
    exe = build.build_tc_test()
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and r.stdout.strip().endswith('OK'), r.stdout + r.stderr


@pytest.mark.parametrize('precision', ['f64', 'f32'])
def test_boundary_repair_cascades_to_the_sequential_result(cases, precision):
    """Chunks with a single warm-up frame (a cold start right in front of the chunk: far off), then the boundary check with
    zero tolerance: every round
    resumes the failing chunks from the rows their predecessors emitted; a resumed chunk whose predecessor is repaired
    later fails the next check (it reports the state it started from).  After at most one round per chunk the result
    is the single sequential pass, bit for bit -- the repair is exact, not an approximation."""
    from moshpp_b200 import chmosh
    case = cases('C2')
    obs, vis = dense_obs(case)
    pk, opts, _ = chmosh.prepare_stageii(case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])
    prec = {'f32': lib.MOSH2_F32, 'f64': lib.MOSH2_F64}[precision]
    model = lib.Model(pk, device=0)
    try:
        seq = model.solve(obs, vis, opts, precision=prec)
        job = model.job(obs.shape[0], opts, chunk_len=3, chunk_warmup=1, precision=prec)
        cold = model.solve(obs, vis, opts, chunk_len=3, chunk_warmup=1, precision=prec)
        assert np.abs(cold.pose - seq.pose).max() > 1e-3
        res, rep = chmosh.solve_verified(job, obs, vis, tol=(0.0, 0.0, 0.0, 0.0), max_rounds=job.num_chunks + 1)
        assert rep['unverified_chunks'] == 0 and 1 <= rep['rounds'] <= job.num_chunks
        assert np.array_equal(res.pose, seq.pose) and np.array_equal(res.trans, seq.trans)
        assert np.array_equal(res.status, seq.status) and np.array_equal(res.errs, seq.errs)
        job.close()
    finally:
        model.close()


def test_drop_in_callable_with_the_horse_model(cases):
    """animal_horse (SURVEY.md 8(f-4); chmosh.py:572-573,615-617): single-Gaussian pose prior + joint-angle term; the return
    dictionary names the term like the reference does."""
    from moshpp_b200.chmosh import mosh_stageii
    case = cases('CH')
    out = mosh_stageii(mocap_fname=case['mocap_fname'], cfg=case['cfg'], markers_latent=case['markers_latent'],
                       latent_labels=case['latent_labels'], betas=case['betas'], marker_meta=case['marker_meta'],
                       precision='f64', chunk_len=0)
    ref = run_oracle(case)
    assert np.abs(out['fullpose'] - ref['fullpose']).max() < 1e-8 and np.abs(out['trans'] - ref['trans']).max() < 1e-9
    e, r = out['stageii_debug_details']['stageii_errs'], ref['stageii_debug_details']['stageii_errs']
    assert set(e.keys()) == set(r.keys()) == {'data', 'poseB', 'poseB_jangles', 'velo'}
    for k in ('data', 'poseB', 'poseB_jangles'):
        assert np.allclose(e[k], r[k], rtol=1e-7, atol=1e-10)
    assert np.abs(out['fullpose'][:, 84:]).max() == 0          # tail, mouth and ears stay at rest


@pytest.mark.parametrize('name', ['C1', 'C2'])
def test_device_input_adapter_equals_host_adapter(cases, name):
    """mosh2_job_upload_markers: the raw marker table of the capture file (c3d in mm for C1, npz for C2; missing samples as
    NaN or zeros; an unknown label; a frame range with a stride; a rotation) turned into observations + visibility on the
    GPU gives bit for bit the result of the host adapter (MocapSession.frames_for_labels) in front of the same solve."""
    import copy
    from moshpp_b200.chmosh import mosh_stageii
    case = cases(name)
    cfg = copy.deepcopy(case['cfg'])
    cfg.mocap.start_fidx, cfg.mocap.end_fidx, cfg.mocap.ds_rate = 1, -1, 2
    cfg.mocap.rotate = [10.0, -20.0, 30.0] if name == 'C2' else None
    args = (case['mocap_fname'], cfg, case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])
    a = mosh_stageii(*args, precision='f32', chunk_len=0, device_adapter=True)
    b = mosh_stageii(*args, precision='f32', chunk_len=0, device_adapter=False)
    assert a['stageii_debug_details']['b200']['device_adapter'] and not b['stageii_debug_details']['b200']['device_adapter']
    da, db = a['stageii_debug_details'], b['stageii_debug_details']
    assert da['labels_obs'] == db['labels_obs']
    assert all(np.array_equal(x, y) for x, y in zip(da['markers_obs'], db['markers_obs']))       # (the host copy of both)
    if cfg.mocap.rotate is None:
        assert np.array_equal(a['fullpose'], b['fullpose']) and np.array_equal(a['trans'], b['trans'])
        assert all(np.array_equal(x, y) for x, y in zip(da['markers_sim'], db['markers_sim']))
    else:       # the rotation is a float64 3x3 product on either side, not necessarily rounded alike in the last bit
        assert np.abs(a['fullpose'] - b['fullpose']).max() < 1e-4 and np.abs(a['trans'] - b['trans']).max() < 1e-5
    assert np.array_equal(da['markers_orig'], db['markers_orig'])
    assert sum(len(l) for l in da['labels_obs']) < len(da['labels_obs']) * len(case['latent_labels'])    # some samples are missing
