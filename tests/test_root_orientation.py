"""CPU suite: Stage II with the body facing any direction and turning through pi.

The sequential pass aligns the first frame of a sequence (Procrustes, an angle in [0, pi]) and then tracks the root as a free
parameter, so a subject who turns past 180 degrees ends up with an axis-angle root beyond pi.  These tests run the device source
(single-thread host build, tests/emu) against the float64 oracle at such roots: the first-frame alignment at any orientation,
the sequential pass across pi, and the chunked schedule, whose chunks align their own first warm-up frame and must be put on
the sequential pass's branch (chmosh.root_branch_turns, the chunk record's root turns).
"""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import dense_obs, run_oracle
from moshpp_b200 import chmosh, lib, synth

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
WINDOW = 48                                   # frames of the short windows the oracle solves live
TURN_WINDOW = (np.pi - 0.3, np.pi + 0.6)      # a turn through pi within the window
BACK_WINDOW = tuple(np.pi + 0.3 * np.sin(2 * np.pi * 3.0 * np.arange(WINDOW) / 120.0 - np.arcsin(1 / 6)))    # facing backwards, swaying


def _emu_turns(emu_handle, case, sched, turns, obs_vis=None):
    pk, cfg = case['pack'], case['cfg']
    obs, vis = obs_vis if obs_vis is not None else dense_obs(case)
    h = lib.DescHolder(pk)
    opt = lib.make_options(cfg.opt_settings.weights, optimize_fingers=cfg.moshpp.optimize_fingers and pk.finger_hi > pk.finger_lo)
    F = obs.shape[0]
    res = lib.ResultArrays(F, lib.pack_dims(pk))
    o = np.ascontiguousarray(obs, dtype=np.float64)
    v8 = np.ascontiguousarray(vis, dtype=np.uint8)
    t = np.ascontiguousarray(turns, dtype=np.int32)
    rc = emu_handle.mosh2_emu_solve_root_turns(C.byref(h.desc), C.byref(opt), F, lib._ptr(o, lib._f64p), lib._ptr(v8, lib._u8p),
                                               C.byref(sched), lib._ptr(t, lib._i32p), lib.MOSH2_F64, C.byref(res.c))
    assert rc == 0
    return res


@pytest.fixture(scope='module')
def emu_handle():
    from moshpp_b200 import build
    return C.CDLL(build.build_emu())


def test_default_motion_is_unchanged():
    """root_yaw is opt-in: without it the random draws and the motion are those every committed fixture was made from."""
    import tempfile
    case = synth.make_case(tempfile.mkdtemp(), 'C2', frames=500)
    gold = np.load(os.path.join(GOLD, 'long_C2.npz'))
    assert np.array_equal(gold['obs_checksum'], [np.nansum(case['obs']), case['vis'].sum()])


def test_root_yaw_composes_a_turn_in_front_of_the_root_motion(cases):
    plain = cases('C2', frames=WINDOW)
    turn = cases('C2', frames=WINDOW, root_yaw=TURN_WINDOW)
    assert plain['mocap_fname'] != turn['mocap_fname']
    yaw = np.linspace(*TURN_WINDOW, WINDOW)
    R = synth.rodrigues_batch(yaw[:, None] * np.array([0.0, 1.0, 0.0])) @ synth.rodrigues_batch(plain['gt_pose'][:, :3])
    assert np.abs(synth.rodrigues_batch(turn['gt_pose'][:, :3]) - R).max() < 1e-12
    assert np.array_equal(turn['gt_pose'][:, 3:], plain['gt_pose'][:, 3:]) and np.array_equal(turn['gt_trans'], plain['gt_trans'])
    th = np.linalg.norm(turn['gt_pose'][:, :3], axis=1)
    assert th[0] < np.pi < th.max()                                     # continuous through pi: unwrapped, not principal
    assert np.abs(np.diff(turn['gt_pose'][:, :3], axis=0)).max() < 0.1


def test_rodrigues_inverse_at_any_angle():
    rng = np.random.default_rng(7)
    ax = rng.standard_normal((400, 3))
    ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    ang = np.concatenate([rng.uniform(0, np.pi, 200), np.pi - np.logspace(-12, -2, 100), rng.uniform(0, 1e-6, 100)])
    rv = ax * ang[:, None]
    back = synth.rodrigues_inv_batch(synth.rodrigues_batch(rv))
    assert np.abs(synth.rodrigues_batch(back) - synth.rodrigues_batch(rv)).max() < 1e-12
    assert (np.linalg.norm(back, axis=1) <= np.pi + 1e-12).all()
    away = ang < np.pi - 1e-6
    assert np.abs(back[away] - rv[away]).max() < 1e-8


def _branch(r, n):
    th = np.linalg.norm(r, axis=-1, keepdims=True)
    return r * (1 + 2 * np.pi * n / th)


def test_root_branch_turns_unwraps_across_chunk_boundaries():
    """chmosh.root_branch_turns on a turn through pi: chunks that emit another branch of the same rotations get the turns
    that put them back on the branch of the chunks in front of them; a new sequence starts over."""
    yaw = np.concatenate([np.linspace(2.6, 3.8, 24), np.linspace(2.9, 3.4, 12)])
    seq = yaw[:, None] * np.array([0.1, 1.0, -0.05]) / np.linalg.norm([0.1, 1.0, -0.05])   # the sequential pass's roots
    ranges = np.array([[0, 6], [6, 12], [12, 18], [18, 24], [24, 30], [30, 36]])
    solved = np.ones(36, dtype=bool)
    emitted = seq.copy()
    emitted[12:18] = _branch(seq[12:18], -1)          # aligned behind the crossing: the principal branch
    emitted[18:24] = _branch(seq[18:24], -1)
    emitted[30:36] = _branch(seq[30:36], -1)          # (second sequence, own start at 24)
    solved[14] = False
    turns = chmosh.root_branch_turns(emitted, solved, ranges, [0, 24])
    assert turns.tolist() == [0, 0, -1, -1, 0, -1]
    assert chmosh.root_branch_turns(seq, solved, ranges, [0, 24]).tolist() == [0] * 6
    # a chunk without a solved frame neither gets turns nor breaks the chain
    solved[6:12] = False
    assert chmosh.root_branch_turns(emitted, solved, ranges, [0, 24]).tolist() == [0, 0, -1, -1, 0, -1]


@pytest.mark.parametrize('which', ['TURN', 'BACK'])
def test_sequential_pass_across_pi_equals_oracle(cases, emu, which):
    """chunk_len = 0 in float64: the root leaves the principal branch exactly where the oracle's does, with the same
    dog-leg path (Jacobian builds) -- Rodrigues and its Jacobian beyond pi."""
    case = cases('C2', frames=WINDOW, root_yaw=TURN_WINDOW if which == 'TURN' else BACK_WINDOW)
    out = run_oracle(case)
    res = emu(case, precision=lib.MOSH2_F64)
    fid = out['stageii_debug_details']['frame_ids']
    ref_root = out['_pose_reduced'][:, :3]
    assert np.linalg.norm(ref_root, axis=1).max() > np.pi + 0.05              # the reference itself goes beyond pi
    assert np.abs(res.pose[fid] - out['_pose_reduced']).max() < 1e-9
    assert np.abs(res.trans[fid] - out['trans']).max() < 1e-10
    assert res.counters[fid, 2].sum() == out['stageii_debug_details']['oracle_stats']['j_evals']


@pytest.mark.parametrize('which', ['TURN', 'BACK'])
def test_chunks_behind_a_pi_crossing_take_the_sequential_branch(cases, emu, emu_handle, which):
    """The chunked schedule in float64: a chunk aligns the first frame of its own warm-up, i.e. lands on the principal
    branch.  Behind a pi crossing that is another axis-angle branch than the sequential pass's -- another problem, since the
    velocity term couples consecutive frames in parameter space.  With the turns chmosh.root_branch_turns derives from the
    first pass, every chunk follows the sequential pass again."""
    case = cases('C2', frames=WINDOW, root_yaw=TURN_WINDOW if which == 'TURN' else BACK_WINDOW)
    seq = emu(case, precision=lib.MOSH2_F64)
    L, W = 4, 16
    sched = lib.make_schedule(L, W, -1)
    ranges = np.array([[f, min(f + L, WINDOW)] for f in range(0, WINDOW, L)])
    first = _emu_turns(emu_handle, case, sched, np.zeros(len(ranges)))
    solved = (first.status & lib.ST_SOLVED) != 0
    assert solved.all()
    jump = np.abs(first.pose[:, :3] - seq.pose[:, :3]).max(1)
    assert jump.max() > 3.0                                                  # (the branch problem: 2 pi apart)
    turns = chmosh.root_branch_turns(first.pose[:, :3], solved, ranges, [0])
    assert (turns != 0).any() and set(np.unique(turns)) <= {-1, 0, 1}
    fixed = _emu_turns(emu_handle, case, sched, turns)
    assert np.array_equal(fixed.pose[turns[np.arange(WINDOW) // L] == 0], first.pose[turns[np.arange(WINDOW) // L] == 0])
    d = np.abs(fixed.pose - seq.pose).max(1)
    assert d.max() < 5e-2, d                                                 # what a 16-frame warm-up leaves, as without a turn
    assert np.abs(np.diff(fixed.pose[:, :3], axis=0)).max() < 0.5


def _first_frame_orientations(seed=11):
    """24 root orientations: uniform random rotations, yaw pi +- {1e-3, 0.05}, angles 3.0..3.14 about random axes, the
    identity."""
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(seed)
    rv = list(Rotation.random(14, random_state=seed).as_rotvec())
    rv += [np.array([0.0, y, 0.0]) for y in (np.pi - 1e-3, np.pi + 1e-3, np.pi - 0.05, np.pi + 0.05)]
    for a in (3.0, 3.07, 3.12, 3.135, 3.14):
        ax = rng.standard_normal(3)
        rv.append(ax / np.linalg.norm(ax) * a)
    rv.append(np.zeros(3))
    return np.array(rv)


def first_frame_case(cases, tmp_dir):
    """48 one-frame captures of one subject: every orientation of _first_frame_orientations with all markers visible and
    with only 3 or 4 of them.  Returns (case with its mocap file replaced, obs, vis, orientations)."""
    base = cases('C2', frames=48)
    pk = base['pack']
    rv = _first_frame_orientations()
    pose = base['gt_pose'].copy()
    pose[:, :3] = np.concatenate([rv, rv])
    mk = synth.forward_markers(pk, pose, base['gt_trans'])
    obs = mk + np.random.default_rng(3).normal(0.0, 1e-3, mk.shape)
    vis = np.ones(obs.shape[:2], dtype=bool)
    rng = np.random.default_rng(4)
    for f in range(24, 48):
        keep = rng.choice(pk.n_markers, 3 + f % 2, replace=False)
        vis[f] = np.isin(np.arange(pk.n_markers), keep)
    labels = list(base['latent_labels'])
    fname = os.path.join(tmp_dir, 'mocap_first_frames_48.npz')
    np.savez(fname, markers=np.where(vis[..., None], obs, np.nan) * 1000.0, labels=np.array(labels), frame_rate=120.0)
    case = dict(base, mocap_fname=fname, obs=obs, vis=vis)
    return case, obs, vis, pose[:, :3]


def root_rotation_errors(got, ref):
    """max |R(got) - R(ref)| per frame, and max |got - ref| per frame away from the tie at pi (the sign of the axis of a
    half-turn is the oracle's choice: within 1e-9 of pi only the rotation is compared)."""
    dR = np.abs(synth.rodrigues_batch(got) - synth.rodrigues_batch(ref)).reshape(len(got), -1).max(1)
    away = np.abs(np.linalg.norm(ref, axis=1) - np.pi) > 1e-9
    drv = np.where(away, np.abs(got - ref).max(1), 0.0)
    return dR, drv


def test_first_frame_at_any_orientation_equals_oracle(cases, case_dir, emu_handle):
    """Every frame a cold start (a batch job of 48 one-frame sequences) against the oracle's first-frame solve (Procrustes +
    the annealed Step-1 minimisations + Steps 1 and 2): Horn's quaternion method with a Jacobi eigen-solve against an SVD
    with the determinant fix and cv2.Rodrigues, far from the identity, near pi and through 3 or 4 markers."""
    case, obs, vis, rv = first_frame_case(cases, case_dir)
    out = run_oracle(case, chunk=(1, 0))                  # every frame solved from its own cold start
    fid = out['stageii_debug_details']['frame_ids']
    assert np.array_equal(fid, np.arange(48))
    pk, cfg = case['pack'], case['cfg']
    h = lib.DescHolder(pk)
    opt = lib.make_options(cfg.opt_settings.weights, optimize_fingers=True)
    res = lib.ResultArrays(48, lib.pack_dims(pk))
    counts = np.ones(48, dtype=np.int32)
    o = np.ascontiguousarray(obs, dtype=np.float64)
    v8 = np.ascontiguousarray(vis, dtype=np.uint8)
    rc = emu_handle.mosh2_emu_solve_batch(C.byref(h.desc), C.byref(opt), 48, lib._ptr(counts, lib._i32p), lib._ptr(o, lib._f64p),
                                          lib._ptr(v8, lib._u8p), C.byref(lib.make_schedule()), lib.MOSH2_F64, C.byref(res.c))
    assert rc == 0
    ref = out['_pose_reduced']
    dR, drv = root_rotation_errors(res.pose[:, :3], ref[:, :3])
    assert dR.max() < 1e-8 and drv.max() < 1e-8
    assert np.abs(res.pose[:, 3:] - ref[:, 3:]).max() < 1e-8
    assert np.abs(res.trans - out['trans']).max() < 1e-8
    assert res.counters[:, 2].sum() == out['stageii_debug_details']['oracle_stats']['j_evals']
    # the alignment found the orientation the captures were made with (all markers visible: within the noise)
    assert (np.abs(synth.rodrigues_batch(ref[:24, :3]) - synth.rodrigues_batch(rv[:24])).reshape(24, -1).max(1) < 0.05).all()
