"""Stage II on the H100 with the body facing any direction and turning through pi, against the float64 oracle.

The CPU twins are in test_root_orientation.py.  The sequential oracle on the two 600-frame SMPL-H captures TURN (the whole
body turns from 2.0 to 5.0 rad about the up axis: its axis-angle root passes pi once) and BACK (it starts facing backwards and
sways around pi, passing it again and again) is committed (tests/golden/long_TURN.npz, long_BACK.npz; make_long_golden.py).
"""
import os

import numpy as np
import pytest

from conftest import run_oracle
from moshpp_b200 import chmosh, lib
from test_gpu_long_parity import GOLD, TOL_BODY, TOL_FINGER, TOL_SSE, TOL_TRANS, _excursions, _full_case, _report, _run_drop_in
from test_root_orientation import first_frame_case, root_rotation_errors

pytestmark = pytest.mark.gpu


def _gold(cases, key):
    case = _full_case(cases, key)
    gold = np.load(os.path.join(GOLD, f'long_{key}.npz'))
    assert np.allclose(gold['obs_checksum'], [np.nansum(case['obs']), case['vis'].sum()], rtol=1e-12)   # same inputs
    return case, gold


def _max_root_step(pose_solved):
    """Largest change of a root component between consecutive solved frames."""
    return np.abs(np.diff(pose_solved[:, :3], axis=0)).max()


@pytest.mark.parametrize('precision', ['f64', 'f32'])
def test_first_frame_at_any_orientation(cases, case_dir, precision):
    """One batch job of 48 one-frame captures of one subject (every frame a cold start: Procrustes, the annealed minimisations,
    Steps 1 and 2) against the oracle's first-frame solve: uniform random orientations, yaw pi +- {1e-3, 0.05}, angles
    3.0..3.14 about random axes and the identity, each with all markers and with 3 or 4 visible."""
    case, obs, vis, _ = first_frame_case(cases, case_dir)
    out = run_oracle(case, chunk=(1, 0))
    ref = out['_pose_reduced']
    pk, opts, _ = chmosh.prepare_stageii(case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])
    model = lib.Model(pk, device=0)
    try:
        job = model.job([1] * 48, opts, precision={'f32': lib.MOSH2_F32, 'f64': lib.MOSH2_F64}[precision])
        try:
            job.upload(obs, vis)
            job.launch()
            res = job.download()
        finally:
            job.close()
    finally:
        model.close()
    assert (res.status & lib.ST_SOLVED).all()
    dR, drv = root_rotation_errors(res.pose[:, :3], ref[:, :3])
    bd = min(pk.body_dof, 66)
    dp = np.abs(res.pose - ref)
    dt = np.abs(res.trans - out['trans']).max(1)
    print(f'\n[first frames {precision}] root rotation max {dR.max():.1e}, root axis-angle max {drv.max():.1e}, body max '
          f'{dp[:, 3:bd].max():.1e} rad, fingers max {dp[:, bd:].max():.1e}, trans max {dt.max():.1e} m')
    if precision == 'f64':
        assert dR.max() < 1e-8 and drv.max() < 1e-8 and dp.max() < 1e-8 and dt.max() < 1e-8
        assert np.array_equal(res.counters[:, 2].sum(), out['stageii_debug_details']['oracle_stats']['j_evals'])
    else:
        # all markers visible: BASELINE.md section 4's tolerances.  Through 3 or 4 markers the body pose rests on the prior
        # alone and the float32 solve is ill-conditioned (the float64 one above matches to 1e-8): there only a bound that a
        # flipped or mis-aligned root (errors of order 1 rad) would break
        full = vis.all(1)
        assert dR[full].max() < TOL_BODY and drv[full].max() < TOL_BODY and dp[full, :bd].max() < TOL_BODY
        assert dp[full, bd:].max() < TOL_FINGER and dt[full].max() < TOL_TRANS
        assert dR.max() < 0.1 and drv.max() < 0.1 and dt.max() < 0.02


@pytest.mark.parametrize('key', ['TURN', 'BACK'])
def test_sequential_f64_across_pi_equals_oracle(cases, key):
    """chunk_len = 0 in float64: the oracle's trajectory -- with its roots beyond pi -- iteration for iteration."""
    case, gold = _gold(cases, key)
    out, b = _run_drop_in(case, chunk_len=0, precision='f64')
    groot = gold['pose'][:, :3].astype(np.float64)
    assert np.linalg.norm(groot, axis=1).max() > np.pi + (1.5 if key == 'TURN' else 0.1)     # the reference leaves the principal branch
    assert np.abs(b['pose_reduced'] - gold['pose']).max() < 1e-6              # fixture stored as float32
    assert np.abs(out['trans'] - gold['trans']).max() < 1e-6
    assert int(b['counters'][:, 2].sum()) == int(gold['j_evals'])


@pytest.mark.parametrize('key', ['TURN', 'BACK'])
def test_default_product_path_across_pi(cases, key):
    """The drop-in callable as shipped (float32, chunked, verified warm-up): chunks that align their warm-up behind a pi
    crossing start on the sequential pass's branch (chmosh.root_branch_turns), so every frame meets the per-frame tolerances
    of test_gpu_long_parity and the root never jumps by a turn."""
    case, gold = _gold(cases, key)
    out, b = _run_drop_in(case)
    bc = b['boundary_check']
    assert b['precision'] == 'f32' and b['chunks'] > 1 and np.array_equal(b['frame_ids'], gold['frame_ids'])
    print(f'\n[{key}] boundary check: rounds {bc["rounds"]}, root-branch chunks {bc.get("root_branch_chunks")}, repaired per round '
          f'{bc["repaired_chunks"]}, first delta {bc["boundary_delta_first"]}, max delta {bc["boundary_delta_max"]}, unverified {bc["unverified_chunks"]}')
    rep = _report(f'{key} default path: chunk_len {b["chunk_len"]}', b['pose_reduced'], out['trans'],
                  out['stageii_debug_details']['stageii_errs']['data'], gold, case['pack'].body_dof)
    assert bc['unverified_chunks'] <= max(1, 0.05 * b['chunks'])
    assert _max_root_step(b['pose_reduced']) < 0.5
    for name, tol in (('body', TOL_BODY), ('finger', TOL_FINGER), ('trans', TOL_TRANS), ('sse', TOL_SSE)):
        over = rep[name] > tol
        runs = _excursions(over)
        assert over.sum() <= 0.01 * len(over), (name, int(over.sum()))
        assert np.sqrt((rep[name] ** 2).mean()) <= tol, name
        assert not runs or max(runs) <= 40, (name, runs)
    assert rep['body'].max() < 0.05 and rep['trans'].max() < 2e-3


@pytest.mark.parametrize('key', ['TURN', 'BACK'])
def test_exact_mode_across_pi(cases, key):
    case, gold = _gold(cases, key)
    out, b = _run_drop_in(case, mode='exact')
    bc = b['boundary_check']
    print(f'\n[{key} exact] rounds {bc["rounds"]}, root-branch chunks {bc.get("root_branch_chunks")}, unverified {bc["unverified_chunks"]}')
    rep = _report(f'{key} exact mode', b['pose_reduced'], out['trans'], out['stageii_debug_details']['stageii_errs']['data'], gold,
                  case['pack'].body_dof)
    assert bc['unverified_chunks'] == 0
    assert rep['body'].max() < 1e-4 and rep['trans'].max() < 1e-5
    assert _max_root_step(b['pose_reduced']) < 0.5


def test_batch_and_subjects_with_turning_captures(cases):
    """A turning capture among others: mosh_stageii_batch, mosh_stageii_subjects and mosh_stageii of each capture on the
    same chunk length return the same rows, bit for bit (the root-branch pass and the repairs work per chunk)."""
    turn, _ = _gold(cases, 'TURN')
    back, _ = _gold(cases, 'BACK')
    plain = _full_case(cases, 'C2')
    fnames = [plain['mocap_fname'], turn['mocap_fname'], back['mocap_fname']]
    args = (turn['cfg'], turn['markers_latent'], turn['latent_labels'], turn['betas'], turn['marker_meta'])
    batch = chmosh.mosh_stageii_batch(fnames, *args)
    L = batch[0]['stageii_debug_details']['b200']['batch']['chunk_len']
    assert batch[1]['stageii_debug_details']['b200']['batch']['boundary_check']['root_branch_chunks'] > 0
    subj = chmosh.mosh_stageii_subjects([dict(cfg=turn['cfg'], mocap_fnames=fnames, markers_latent=turn['markers_latent'],
                                              latent_labels=turn['latent_labels'], betas=turn['betas'],
                                              marker_meta=turn['marker_meta'])], chunk_len=L)[0]
    for q, fn in enumerate(fnames):
        single = chmosh.mosh_stageii(fn, *args, chunk_len=L)
        for other in (subj[q], single):
            for k in ('fullpose', 'trans'):
                assert np.array_equal(batch[q][k], other[k]), (q, k)
            assert np.array_equal(batch[q]['stageii_debug_details']['b200']['status'], other['stageii_debug_details']['b200']['status'])
