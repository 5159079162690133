"""CPU suite: the device source (single-thread host build, tests/emu) against the float64 oracle.

This validates index math and control flow of the exact code nvcc compiles; the numbers that count are
the `-m gpu` twins in test_gpu_parity.py, which call the CUDA library through the C-ABI.
"""
import dataclasses

import numpy as np
import pytest

from conftest import run_oracle
from moshpp_b200 import lib


@pytest.mark.parametrize('name', ['C1', 'C2', 'C3', 'C4', 'CF', 'CH', 'C2-kw5'])
def test_f64_device_source_equals_oracle(cases, emu, name):
    case = cases(name.split('-')[0])
    if name.endswith('-kw5'):
        # the same model with an empty fifth skinning column (joint -1, weight 0): the Jacobian takes the generic
        # per-joint skinning loop instead of the four-joint vector path of the released models
        pk = case['pack']
        assert pk.kw == 4
        case = dict(case, pack=dataclasses.replace(pk, kw=5, w_joint=np.pad(pk.w_joint, ((0, 0), (0, 1)), constant_values=-1),
                                                   w_val=np.pad(pk.w_val, ((0, 0), (0, 1)))))
    out = run_oracle(case)
    res = emu(case, precision=lib.MOSH2_F64)
    dbg = out['stageii_debug_details']
    fid = dbg['frame_ids']
    assert np.array_equal(np.nonzero(res.status & lib.ST_SOLVED)[0], fid)
    assert np.abs(res.pose[fid] - out['_pose_reduced']).max() < 1e-9
    assert np.abs(res.fullpose[fid] - out['fullpose']).max() < 1e-9
    assert np.abs(res.trans[fid] - out['trans']).max() < 1e-10
    if 'dmpls' in out:
        assert np.abs(res.dmpls[fid, :out['dmpls'].shape[1]] - out['dmpls']).max() < 1e-9
    if 'expression' in out:                      # the expression coefficients are the tail of the linear block
        pk = case['pack']
        assert pk.n_expr > 0 and np.abs(out['expression'][:, :pk.n_expr]).max() > 1e-2
        assert np.abs(res.dmpls[fid, pk.n_dmpl - pk.n_expr:pk.n_dmpl] - out['expression'][:, :pk.n_expr]).max() < 1e-9
    # identical dog-leg trajectories: same number of Jacobian builds and minimisations
    assert res.counters[fid, 2].sum() == dbg['oracle_stats']['j_evals']
    assert res.counters[fid, 3].sum() == dbg['oracle_stats']['minimizations']
    for col, k in enumerate(lib.ERR_NAMES):
        if k in dbg['stageii_errs'] and k not in ('velo', 'extrap_dmpl'):
            assert np.allclose(res.errs[fid, col], dbg['stageii_errs'][k], rtol=1e-8, atol=1e-12)
    if 'poseB_jangles' in dbg['stageii_errs']:          # animal_horse: the joint-angle term is reported in the poseH column
        assert np.allclose(res.errs[fid, lib.ERR_NAMES.index('poseH')], dbg['stageii_errs']['poseB_jangles'], rtol=1e-8, atol=1e-12)
        assert dbg['stageii_errs']['poseB_jangles'].min() > 0
    n_velo = int(((res.status[fid] & lib.ST_HAS_VELO) != 0).sum())
    assert n_velo == len(dbg['stageii_errs'].get('velo', []))


def test_f32_device_source_within_tolerance(cases, emu):
    case = cases('C2')
    out = run_oracle(case)
    res = emu(case, precision=lib.MOSH2_F32)
    fid = out['stageii_debug_details']['frame_ids']
    bd = case['pack'].body_dof
    dp = np.abs(res.pose[fid] - out['_pose_reduced'])
    assert dp[:, :bd].max() < 1e-3          # body pose, rad
    assert dp.max() < 5e-3                   # weakly observed finger PCA coefficients
    assert np.abs(res.trans[fid] - out['trans']).max() < 1e-4
    sse = out['stageii_debug_details']['stageii_errs']['data']
    assert np.abs(res.errs[fid, 0] / sse - 1).max() < 1e-2


def test_chunked_schedule_matches_oracle_chunked(cases, emu):
    case = cases('C2')
    out = run_oracle(case, chunk=(5, 2))
    res = emu(case, chunk_len=5, warmup=2)
    fid = out['stageii_debug_details']['frame_ids']
    assert np.abs(res.pose[fid] - out['_pose_reduced']).max() < 1e-9


def test_chunk_warmup_converges_to_sequential(cases, emu):
    """The reference recursion is contractive: chunks started W frames early converge to the single
    sequential pass geometrically in W (DESIGN.md section 4)."""
    case = cases('C2', frames=160)
    seq = emu(case)
    ok = (seq.status & lib.ST_SOLVED) != 0
    errs = []
    for W in (0, 16, 48, 96):
        ch = emu(case, chunk_len=32, warmup=W)
        errs.append(np.abs(ch.pose - seq.pose)[ok].max())
    assert errs[1] < 0.5 * errs[0] and errs[2] < 1e-3 and errs[3] < 1e-6, errs


def test_frames_without_markers_are_skipped(cases, emu):
    case = cases('C1')
    from conftest import dense_obs
    obs, vis = dense_obs(case)
    vis = vis.copy()
    vis[3] = False
    vis[7] = False
    res = emu(case, obs_vis=(obs, vis))
    assert res.status[3] == lib.ST_SKIPPED and res.status[7] == lib.ST_SKIPPED
    assert (res.status[[0, 1, 2, 4]] & lib.ST_SOLVED).all()
    # velocity term needs two processed predecessors (chmosh.py:624-626,656-657)
    assert not (res.status[0] & lib.ST_HAS_VELO) and not (res.status[1] & lib.ST_HAS_VELO)
    assert res.status[2] & lib.ST_HAS_VELO and res.status[4] & lib.ST_HAS_VELO


def test_light_warmup_schedule_matches_oracle_emulation(cases, emu):
    """Chunks with a light warm-up (one Step-2 iteration per frame) followed by fully solved warm-up frames: the device
    source against the oracle's independent emulation of the same schedule, incl. frames without markers inside the
    warm-up window (the warm-up is counted in solved frames)."""
    from conftest import dense_obs
    case = cases('C2')
    obs, vis = dense_obs(case)
    vis = vis.copy()
    vis[6] = False
    vis[7] = False
    from oracle import stageii
    from moshpp_b200.mocap_interface import MocapSession
    mocap = MocapSession(case['mocap_fname'], case['cfg'].mocap.unit)
    mocap.markers[6:8] = 0.0
    out = stageii.mosh_stageii(case['mocap_fname'], case['cfg'], case['markers_latent'], case['latent_labels'],
                               case['betas'], case['marker_meta'], chunk=(4, 5, 2), mocap=mocap)
    res = emu(case, chunk_len=4, warmup=5, warmup_full=2, obs_vis=(obs, vis))
    fid = out['stageii_debug_details']['frame_ids']
    assert 6 not in fid and res.status[6] == lib.ST_SKIPPED
    assert np.abs(res.pose[fid] - out['_pose_reduced']).max() < 1e-9
    # not the same numbers as with a fully solved warm-up
    full = emu(case, chunk_len=4, warmup=5, obs_vis=(obs, vis))
    assert np.abs(full.pose[fid] - res.pose[fid]).max() > 1e-6


def test_batch_job_equals_separate_sequences(cases, emu):
    """mosh2_job_create_batch: several sequences of one subject back to back on the job's frame axis.  Every sequence
    starts from its own cold start, chunks and their warm-up never reach across a sequence boundary: the rows of each
    sequence equal those of the sequence solved on its own, in the sequential and in the chunked schedule."""
    import ctypes as C
    from conftest import dense_obs
    from moshpp_b200 import build
    case = cases('C2')
    obs, vis = dense_obs(case)
    counts = np.array([7, 9], dtype=np.int32)                     # 16 frames cut into two "sequences"
    handle = C.CDLL(build.build_emu())
    pk, cfg = case['pack'], case['cfg']
    h = lib.DescHolder(pk)
    opt = lib.make_options(cfg.opt_settings.weights, optimize_fingers=True)
    o = np.ascontiguousarray(obs, dtype=np.float64)
    v8 = np.ascontiguousarray(vis, dtype=np.uint8)
    for L, W, WF in ((0, 0, -1), (3, 4, 2)):
        sched = lib.make_schedule(L, W, WF)
        res = lib.ResultArrays(16, lib.pack_dims(pk))
        rc = handle.mosh2_emu_solve_batch(C.byref(h.desc), C.byref(opt), 2, counts.ctypes.data_as(lib._i32p),
                                          o.ctypes.data_as(lib._f64p), v8.ctypes.data_as(lib._u8p), C.byref(sched),
                                          lib.MOSH2_F64, C.byref(res.c))
        assert rc == 0
        a = emu(case, chunk_len=L, warmup=W, warmup_full=WF, obs_vis=(obs[:7], vis[:7]))
        b = emu(case, chunk_len=L, warmup=W, warmup_full=WF, obs_vis=(obs[7:], vis[7:]))
        assert np.array_equal(res.pose[:7], a.pose) and np.array_equal(res.pose[7:], b.pose)
        assert np.array_equal(res.status[:7], a.status) and np.array_equal(res.status[7:], b.status)
        assert not (res.status[7] & lib.ST_HAS_VELO)              # the second sequence starts cold


@pytest.mark.parametrize('name', ['C2', 'C3'])
def test_resumed_chunks_continue_the_sequential_recursion(cases, emu, name):
    """Boundary repair (mosh2_job_relaunch_chunks, chunk_warmup < 0): a chunk that resumes from the rows the previous
    chunk emitted goes on exactly as that chunk would have.  Cold-started chunks without any warm-up, then every chunk
    resumed in order, therefore reproduce the single sequential pass bit for bit -- pose, velocity term, DMPL terms."""
    import ctypes as C
    from conftest import dense_obs
    from moshpp_b200 import build
    case = cases(name)
    obs, vis = dense_obs(case)
    vis = vis.copy()
    vis[5] = False                               # a skipped frame right before a chunk boundary
    seq = emu(case, obs_vis=(obs, vis))
    cold = emu(case, chunk_len=3, warmup=0, obs_vis=(obs, vis))
    assert np.abs(cold.pose - seq.pose).max() > 1e-4
    handle = C.CDLL(build.build_emu())
    pk, cfg = case['pack'], case['cfg']
    h = lib.DescHolder(pk)
    opt = lib.make_options(cfg.opt_settings.weights, optimize_fingers=cfg.moshpp.optimize_fingers and pk.finger_hi > pk.finger_lo,
                           optimize_dynamics=cfg.moshpp.optimize_dynamics)
    F = obs.shape[0]
    res = lib.ResultArrays(F, lib.pack_dims(pk))
    o = np.ascontiguousarray(obs, dtype=np.float64)
    v8 = np.ascontiguousarray(vis, dtype=np.uint8)
    sched = lib.make_schedule(3, 0, -1)
    rc = handle.mosh2_emu_solve_resumed(C.byref(h.desc), C.byref(opt), F, o.ctypes.data_as(lib._f64p), v8.ctypes.data_as(lib._u8p),
                                        C.byref(sched), lib.MOSH2_F64, C.byref(res.c))
    assert rc == 0
    assert np.array_equal(res.status, seq.status)
    assert np.array_equal(res.pose, seq.pose) and np.array_equal(res.trans, seq.trans) and np.array_equal(res.errs, seq.errs)
    if pk.n_dmpl:
        assert np.array_equal(res.dmpls, seq.dmpls)


def test_rank_deficient_frames_are_flagged_and_recovered(cases, emu):
    """A first frame seen through one marker (and a second through two) leaves the root orientation unobserved: the
    Gauss-Newton system is numerically singular.  chumpy solves such a system with LU / lstsq (an arbitrary null-space
    component, clipped by the trust region: there is no result to be faithful to); the kernel's Cholesky declares it
    not positive definite, takes the Cauchy step and says so (MOSH2_ST_GN_FALLBACK).  Both stay finite, and once the
    markers are back the recursion pulls the two solutions together again."""
    from conftest import dense_obs
    from moshpp_b200.mocap_interface import MocapSession
    from oracle import stageii
    case = cases('C1')
    obs, vis = dense_obs(case)
    vis = vis.copy()
    vis[0, 1:] = False
    vis[1, 2:] = False
    res = emu(case, obs_vis=(obs, vis))
    assert (res.status[:2] & lib.ST_GN_FALLBACK).all() and not (res.status[2:] & lib.ST_GN_FALLBACK).any()
    assert (res.status & lib.ST_SOLVED).all() and np.isfinite(res.pose).all() and np.isfinite(res.errs).all()
    mocap = MocapSession(case['mocap_fname'], case['cfg'].mocap.unit)
    col = {l: i for i, l in enumerate(mocap.labels)}
    for f, keep in ((0, 1), (1, 2)):
        for l in case['latent_labels'][keep:]:
            mocap.markers[f, col[l]] = 0.0
    ref = stageii.mosh_stageii(case['mocap_fname'], case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'],
                               case['marker_meta'], mocap=mocap)
    d = np.abs(res.pose - ref['_pose_reduced']).max(1)
    sse = ref['stageii_debug_details']['stageii_errs']['data']
    assert d[-1] < 0.1 * d[2] or d[-1] < 1e-2                  # the difference decays once all markers are seen
    assert np.abs(res.errs[-3:, 0] / sse[-3:] - 1).max() < 0.05


def test_chunks_that_reach_the_sequence_start_are_exact(cases, emu):
    """A chunk whose warm-up walk-back runs into the first frame of the sequence solves those frames fully: it is the
    reference's own recursion from its own start, so its rows equal the single sequential pass bit for bit.  The first
    chunk with a complete warm-up window keeps its light frames."""
    case = cases('C2')
    seq = emu(case)
    res = emu(case, chunk_len=4, warmup=12, warmup_full=8)
    assert np.array_equal(res.pose[:12], seq.pose[:12]) and np.array_equal(res.trans[:12], seq.trans[:12])
    assert np.array_equal(res.errs[:12], seq.errs[:12])
    d = np.abs(res.pose[12:] - seq.pose[12:]).max()
    assert 0 < d < 1e-1


def test_longer_first_chunk_schedule(cases, emu):
    """mosh2_schedule.first_extra: the first chunk of a sequence (no warm-up to solve) emits chunk_len + first_extra frames.
    Its rows are the sequential pass bit for bit; the later chunks follow the oracle's emulation of the same schedule."""
    case = cases('C2')
    seq = emu(case)
    res = emu(case, chunk_len=3, warmup=5, warmup_full=3, first_extra=4)
    assert np.array_equal(res.pose[:7], seq.pose[:7]) and np.array_equal(res.errs[:7], seq.errs[:7])
    assert (res.status & lib.ST_SOLVED).all()
    out = run_oracle(case, chunk=(3, 5, 3, 4))
    assert np.abs(res.pose - out['_pose_reduced']).max() < 1e-9
    assert np.abs(res.trans - out['trans']).max() < 1e-9
    plain = emu(case, chunk_len=3, warmup=5, warmup_full=3)
    assert np.abs(plain.pose[7:] - res.pose[7:]).max() > 1e-9            # other chunk boundaries, other warm-up windows
