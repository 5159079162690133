"""The product path as shipped and timed -- float32, chunked in time with the default warm-up, through the drop-in
callable ``chmosh.mosh_stageii`` -- against the SEQUENTIAL float64 oracle on the BASELINE configurations at full size.

The oracle outputs are committed fixtures (tests/golden/long_*.npz, generator make_long_golden.py: the frame-serial
numpy solve takes minutes, the GPU box only re-creates the seeded inputs).  Tolerances are BASELINE.md section 4's, per
frame; every test prints how many frames exceed each tolerance and the worst frame, and asserts none does.
"""
import os

import numpy as np
import pytest

from conftest import dense_obs
from moshpp_b200 import lib

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')

TOL_BODY, TOL_FINGER, TOL_TRANS, TOL_SSE = 1e-3, 1e-2, 1e-4, 1e-2     # rad, PCA coefficient, m, relative


def _full_case(cases, key):
    import sys
    sys.path.insert(0, GOLD)
    from make_long_golden import LONG
    name, kw = LONG[key]
    return cases(name, n_verts=None, **kw)


def _report(tag, pose, trans, sse, gold, body_dof, tol_body=TOL_BODY):
    """Per-frame deviations from the fixture; returns the dict the assertions use and prints the summary.  (The
    fixtures of the 4000-frame sequences hold the poses of their first solved frames only: make_long_golden.POSE_FRAMES.)"""
    fid = gold['frame_ids']
    npose = len(gold['pose'])
    dp = np.abs(pose[:npose] - gold['pose'].astype(np.float64))
    bd = min(body_dof, 66)
    body = dp[:, :bd].max(1)
    finger = dp[:, bd:].max(1) if dp.shape[1] > bd else np.zeros(len(dp))
    dtr = np.abs(trans - gold['trans'].astype(np.float64)).max(1)
    dsse = np.abs(sse / gold['err_data'] - 1)
    rep = dict(n=len(fid), body=body, finger=finger, trans=dtr, sse=dsse)
    print(f'\n[{tag}] {len(fid)} frames vs sequential float64 oracle:')
    for name, v, tol, unit in (('root+body pose', body, tol_body, 'rad'), ('finger PCA', finger, TOL_FINGER, ''),
                               ('trans', dtr, TOL_TRANS, 'm'), ('data SSE (rel)', dsse, TOL_SSE, '')):
        w = int(np.argmax(v))
        print(f'    {name:15s} max {v.max():.2e} {unit} (frame {int(fid[w])}), rms {np.sqrt((v ** 2).mean()):.1e}, '
              f'frames over {tol:g}: {int((v > tol).sum())} ({100.0 * (v > tol).mean():.2f} %)')
    return rep


def _run_drop_in(case, **kw):
    from moshpp_b200.chmosh import mosh_stageii
    out = mosh_stageii(mocap_fname=case['mocap_fname'], cfg=case['cfg'], markers_latent=case['markers_latent'],
                       latent_labels=case['latent_labels'], betas=case['betas'], marker_meta=case['marker_meta'],
                       v_template_fname=None, **kw)
    b = out['stageii_debug_details']['b200']
    return out, b


def _excursions(over):
    """Lengths of the runs of consecutive frames over tolerance."""
    runs, n = [], 0
    for o in over:
        if o:
            n += 1
        elif n:
            runs.append(n)
            n = 0
    if n:
        runs.append(n)
    return runs


# The reference's sequential result is ill-conditioned on a few frames per thousand: the dog-leg takes discrete decisions
# (accept / reject, trust-region update, the 1 % stop rule, the arg-min component of the max-mixture prior), and on such a
# frame a perturbation of the OBSERVATIONS by 1e-6 m -- a thousandth of the marker noise -- moves the float64 oracle's own
# pose by 5e-3 rad, decaying over the next ~15 frames (tools/oracle_sensitivity.py, BASELINE.md section 4).  No float32
# solve and no time-parallel schedule can follow the reference through those frames; the fast mode's parity statement is
# therefore per frame for >= 99 % of the frames plus bounded, short excursions, and the exact mode (float64) covers all.
@pytest.mark.parametrize('key,kw,tol_body,max_over', [
    ('C2', {}, TOL_BODY, 0.0),                       # BASELINE configs[1]: 500 frames -> chunks of 4
    ('NS', {}, TOL_BODY, 0.01),                      # north-star target: 4000-frame SMPL-H -> chunks of 30
    ('C3', dict(chunk_len=28), 1e-4, 0.0),           # 640-frame window of configs[2], cut with the chunk length of 4000 frames
    ('C3F', {}, 1e-4, 0.0),                          # configs[2] in full: SMPL-X + DMPL, 4000 frames (default: the exact preset)
    ('C4L', {}, 5e-3, 0.01),                         # configs[3]: hand-only model, the wrist is weakly observed (BASELINE.md 4)
    ('C4R', {}, 5e-3, 0.01),
])
def test_default_product_path_vs_sequential_oracle(cases, key, kw, tol_body, max_over):
    case = _full_case(cases, key)
    gold = np.load(os.path.join(GOLD, f'long_{key}.npz'))
    assert np.allclose(gold['obs_checksum'], [np.nansum(case['obs']), case['vis'].sum()], rtol=1e-12)   # same inputs
    out, b = _run_drop_in(case, **kw)
    # the product path: float32 for the body models without per-frame linear coefficients; float64 with DMPL (BASELINE
    # config 3: float32 left the tolerance on 7 % of its frames) and for the hand-only MANO model (chmosh.default_schedule)
    assert b['precision'] == ('f64' if key.startswith(('C4', 'C3')) else 'f32') and b['mode'] == 'fast' and b['chunk_len'] > 0 and b['chunks'] > 1
    assert np.array_equal(b['frame_ids'], gold['frame_ids'])
    bc = b['boundary_check']
    print(f'\n[{key}] boundary check: rounds {bc["rounds"]}, chunks over tolerance at first {bc.get("chunks_over_tol_first")}, repaired per round {bc["repaired_chunks"]}, first delta {bc["boundary_delta_first"]}, max delta {bc["boundary_delta_max"]}, '
          f'unverified {bc["unverified_chunks"]}; executed / useful frame-iterations {b["totals"]["builds"]} / {b["totals"]["emitted_builds"]}')
    rep = _report(f'{key} default path: chunk_len {b["chunk_len"]}, warm-up {b["chunk_warmup"]} ({b["warmup_full"]} full)',
                  b['pose_reduced'], out['trans'], out['stageii_debug_details']['stageii_errs']['data'], gold,
                  case['pack'].body_dof, tol_body)
    if 'dmpls' in gold.files:
        dd = np.abs(out['dmpls'][:len(gold['dmpls'])] - gold['dmpls']).max(1)
        print(f'    dmpl coefficients max {dd.max():.2e}, frames over 1e-2: {(dd > 1e-2).sum()}')
    st = b['status']
    assert not (st & (lib.ST_GN_FALLBACK | lib.ST_MAXITER)).any()
    # a chunk boundary next to an ill-conditioned frame cannot be verified by any warm-up (both sides sit on different
    # branches of the reference's own decision); such chunks stay flagged
    assert bc['unverified_chunks'] <= max(1, 0.05 * b['chunks'])
    assert int(((st & lib.ST_SHORT_WARMUP) != 0).sum()) <= bc['unverified_chunks'] * b['chunk_len']
    for name, tol in (('body', tol_body), ('finger', TOL_FINGER), ('trans', TOL_TRANS), ('sse', TOL_SSE)):
        over = rep[name] > tol
        n = len(over)
        runs = _excursions(over)
        assert over.sum() <= max_over * n, (name, int(over.sum()), n)
        assert np.sqrt((rep[name] ** 2).mean()) <= tol, name                       # typical frame: well inside
        assert not runs or max(runs) <= 40, (name, runs)                            # excursions are short: they decay
    assert rep['body'].max() < 0.05 and rep['trans'].max() < 2e-3                    # and bounded
    if 'markers_sim' in gold.files and max_over == 0.0:
        mk = np.concatenate(out['stageii_debug_details']['markers_sim'])
        assert np.abs(mk - gold['markers_sim']).max() < 1e-4


@pytest.mark.parametrize('key,kw', [('NS', {}), ('C3', dict(chunk_len=28)), ('C4L', {})])
def test_exact_mode_vs_sequential_oracle(cases, key, kw):
    """mode='exact' (float64, 256 fully solved warm-up frames, tight boundary check): every frame of the chunked solve
    on the reference's own sequential float64 result."""
    case = _full_case(cases, key)
    gold = np.load(os.path.join(GOLD, f'long_{key}.npz'))
    out, b = _run_drop_in(case, mode='exact', **kw)
    assert b['precision'] == 'f64' and b['chunks'] > 1
    bc = b['boundary_check']
    print(f'\n[{key} exact] kernel {b["kernel_ms"]:.1f} ms, boundary check: rounds {bc["rounds"]}, repaired per round {bc["repaired_chunks"]}, '
          f'max delta {bc["boundary_delta_max"]}, unverified {bc["unverified_chunks"]}')
    rep = _report(f'{key} exact mode: chunk_len {b["chunk_len"]}, warm-up {b["chunk_warmup"]}', b['pose_reduced'], out['trans'],
                  out['stageii_debug_details']['stageii_errs']['data'], gold, case['pack'].body_dof)
    assert bc['unverified_chunks'] == 0
    # (the fixtures hold float32 copies of the oracle's poses: 6e-8)
    assert rep['body'].max() < 1e-4 and rep['finger'].max() < 1e-3 and rep['trans'].max() < 1e-5 and rep['sse'].max() < 1e-3
    assert abs(int(b['counters'][b['frame_ids'], 2].sum()) - int(gold['j_evals'])) <= 2


def test_sequential_f32_kernel_vs_oracle_on_a_long_sequence(cases):
    """chunk_len = 0 (one thread block, the reference's recursion) in float32 over 500 frames: round-off does not
    accumulate along the sequence."""
    case = _full_case(cases, 'C2')
    gold = np.load(os.path.join(GOLD, 'long_C2.npz'))
    out, b = _run_drop_in(case, chunk_len=0)
    rep = _report('C2 sequential f32', b['pose_reduced'], out['trans'], out['stageii_debug_details']['stageii_errs']['data'],
                  gold, case['pack'].body_dof)
    assert (rep['body'] <= TOL_BODY).all() and (rep['finger'] <= TOL_FINGER).all() and (rep['trans'] <= TOL_TRANS).all()
    # float64 in the same mode reproduces the oracle's dog-leg path iteration for iteration
    out64, b64 = _run_drop_in(case, chunk_len=0, precision='f64')
    assert int(b64['counters'][:, 2].sum()) == int(gold['j_evals'])
    assert np.abs(b64['pose_reduced'] - gold['pose']).max() < 1e-6          # fixture stored as float32


def test_occlusion_gap_across_chunk_boundaries(cases):
    """30 frames without any marker (skipped, chmosh.py:586-588) framed by 10 + 10 frames with three markers only
    (annealed prior weights): the warm-up is counted in solved frames, so the chunks behind the gap carry the pose
    across it like the sequential pass does."""
    import sys
    sys.path.insert(0, GOLD)
    from make_long_golden import blank_gap
    case = _full_case(cases, 'GAP')
    gold = np.load(os.path.join(GOLD, 'long_GAP.npz'))
    mocap = blank_gap(case)
    obs, vis = mocap.frames_for_labels(case['latent_labels'], range(len(mocap)))
    from moshpp_b200 import chmosh
    pk, opts, flags = chmosh.prepare_stageii(case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'],
                                             case['marker_meta'])
    model = lib.Model(pk, device=0)
    try:
        res = model.solve(obs, vis, opts, chunk_len=4, chunk_warmup=chmosh.DEFAULT_WARMUP,
                          warmup_full=chmosh.DEFAULT_WARMUP_FULL, precision=lib.MOSH2_F32)
    finally:
        model.close()
    fid = gold['frame_ids']
    assert np.array_equal(np.nonzero(res.status & lib.ST_SOLVED)[0], fid)
    assert (res.status[100:130] == lib.ST_SKIPPED).all()
    assert not (res.status & lib.ST_SHORT_WARMUP).any()
    rep = _report('GAP chunked f32', res.pose[fid], res.trans[fid], res.errs[fid, 0], gold, pk.body_dof)
    # frames seen through three markers are held by the priors and the velocity term: loosely determined, so the
    # comparison there is on the well-observed frames; behind the gap (frames 140..) the tolerances hold again
    well = np.isin(fid, np.r_[0:90, 140:240])
    assert (rep['body'][well] <= TOL_BODY).all() and (rep['trans'][well] <= TOL_TRANS).all()
    assert rep['body'].max() < 5e-2       # (frames 130..139: three markers, held by priors and velocity only)


def test_c5_shaped_sharded_solve(cases):
    """BASELINE configs[4] in small: four SMPL-H sequences through shard.solve_sharded (scatter -> this rank's GPU solver
    with device-pointer upload / download -> gather) on a one-rank NCCL group, against the sequential oracle."""
    import socket

    import torch
    import torch.distributed as dist

    from moshpp_b200 import chmosh, shard
    keys = ['C5a', 'C5b', 'C5c', 'C5d']
    cs = [_full_case(cases, k) for k in keys]
    golds = [np.load(os.path.join(GOLD, f'long_{k}.npz')) for k in keys]
    with socket.socket() as sk:
        sk.bind(('127.0.0.1', 0))
        port = sk.getsockname()[1]
    os.environ['MASTER_ADDR'], os.environ['MASTER_PORT'] = '127.0.0.1', str(port)
    torch.cuda.set_device(0)
    dist.init_process_group('nccl', rank=0, world_size=1, device_id=torch.device('cuda', 0))
    try:
        packs, obs_list, vis_list, opts = {}, [], [], None
        for i, c in enumerate(cs):
            pk, opts, _ = chmosh.prepare_stageii(c['cfg'], c['markers_latent'], c['latent_labels'], c['betas'], c['marker_meta'])
            packs[i] = pk
            o, v = dense_obs(c)
            obs_list.append(torch.from_numpy(o.astype(np.float32)).pin_memory())
            vis_list.append(torch.from_numpy(v.astype(np.uint8)).pin_memory())
        F = [o.shape[0] for o in obs_list]
        solver = shard.GpuRankSolver(packs, opts, dict(enumerate(F)), 0, chunk_warmup=chmosh.DEFAULT_WARMUP,
                                     warmup_full=chmosh.DEFAULT_WARMUP_FULL)
        width = solver.row_width
        out, assignment = shard.solve_sharded(F, [packs[i].n_markers for i in range(4)], [width] * 4, solver, obs_list, vis_list)
        assert assignment == [[0, 1, 2, 3]] and sorted(out) == [0, 1, 2, 3]
        for i, (c, g) in enumerate(zip(cs, golds)):
            rows = out[i].cpu().numpy().astype(np.float64)
            pk = packs[i]
            PF = 3 * pk.n_joints
            fullpose, trans, errs, status = rows[:, :PF], rows[:, PF:PF + 3], rows[:, PF + 3:PF + 11], rows[:, PF + 11].astype(int)
            fid = g['frame_ids']
            assert np.array_equal(np.nonzero(status & lib.ST_SOLVED)[0], fid)
            # the fixture holds the reduced pose; expand it (smpl_fast_derivatives.py:194-204)
            gp = g['pose'].astype(np.float64)
            gfull = np.concatenate([gp[:, :pk.body_dof], pk.hands_mean[None] + gp[:, pk.body_dof:] @ pk.hand_comps], 1)
            d = np.abs(fullpose[fid] - gfull)
            print(f'\n[C5 seq {i}] chunk_len {solver.chunk_len}: body max {d[:, :66].max():.2e} rad, '
                  f'hands max {d[:, 66:].max():.2e} rad, trans max {np.abs(trans[fid] - g["trans"]).max():.2e} m')
            body = d[:, :66].max(1)
            assert (body > TOL_BODY).mean() <= 0.03 and np.sqrt((body ** 2).mean()) < TOL_BODY and body.max() < 0.05
            assert (np.abs(trans[fid] - g['trans']).max(1) > TOL_TRANS).mean() <= 0.03
            assert (np.abs(errs[fid, 0] / g['err_data'] - 1) > TOL_SSE).mean() <= 0.03
        solver.close()
    finally:
        dist.destroy_process_group()
