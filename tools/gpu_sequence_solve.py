"""The joint minimisation of the sequence objective (``sequence_sweeps``) on one GPU, on the 4000-frame north-star SMPL-H
capture (BASELINE config 5 shape) and the C3 capture, each in its default mode.

Reported per capture: the device time of the causal solve (verified launch, repairs included), the sweeps run and whether
they converged (the mode's ``BOUNDARY_TOL``), the device time per sweep, S of the causal and of the joint result, and the
root + body pose error against the synthetic ground truth over all frames, over the 30 cold first frames and over the 30
frames after each marker dropout.  The dropouts are made here: every marker of ``--dropout`` frames is removed at five places
of each capture (the synthetic captures have none of their own).  Prints one JSON line with the card's name and power limit; ``--out`` also writes it.

    python tools/gpu_sequence_solve.py --sweeps 64 --out seq.json
"""
import argparse
import copy
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f'unknown ({e})'


def after_dropouts(status_solved, n=30):
    """Processed frames within n processed frames after a skipped frame."""
    mark = np.zeros(len(status_solved), dtype=bool)
    gap, left = False, 0
    for f, ok in enumerate(status_solved):
        if not ok:
            gap = True
            continue
        if gap:
            left, gap = n, False
        if left > 0:
            mark[f] = True
            left -= 1
    return mark[status_solved]


def with_dropouts(case, length, d):
    """The case's capture with every marker of ``length`` frames removed at five evenly spaced places, written as an npz mocap
    file (millimetres, missing = NaN); returns its cfg."""
    from bench import dense
    obs, vis = dense(case)
    vis = vis.copy()
    F = len(obs)
    for k in range(1, 6):
        a = k * F // 6
        vis[a:a + length] = False
    fn = os.path.join(d, 'dropouts.npz')
    np.savez(fn, markers=np.where(vis[..., None], obs, np.nan) * 1000.0, labels=np.array(case['latent_labels']), frame_rate=120.0)
    cfg = copy.deepcopy(case['cfg'])
    cfg.mocap.fname = fn
    return fn, cfg


def run(name, sweeps, dropout, d):
    from bench import make_case
    from moshpp_b200 import chmosh
    case = make_case(name, 0, tag='seq_')
    fn, cfg = with_dropouts(case, dropout, d) if dropout > 0 else (case['mocap_fname'], case['cfg'])
    args = (fn, cfg, case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])
    causal = chmosh.mosh_stageii(*args)                      # (warms the subject cache and the kernels)
    causal = chmosh.mosh_stageii(*args)
    joint = chmosh.mosh_stageii(*args, sequence_sweeps=sweeps)
    out = dict(frames=int(len(case['obs'])))
    bc, bj = causal['stageii_debug_details']['b200'], joint['stageii_debug_details']['b200']
    rec = bj['sequence_solve']
    fid = bc['frame_ids']
    solved = np.zeros(out['frames'], dtype=bool)
    solved[fid] = True
    nb = min(int(case['pack'].body_dof), 66)             # root + body pose: the same coefficients in the full and reduced pose
    gt = np.asarray(case['gt_pose']).reshape(out['frames'], -1)[fid][:, :nb]
    near = after_dropouts(solved)
    for k, b in (('causal', bc), ('joint', bj)):
        e = np.abs(b['pose_reduced'][:, :nb] - gt)
        out[k] = dict(max_rad=float(e.max()), mean_rad=float(e.mean()),
                      first30_max_rad=float(e[:30].max()), first30_mean_rad=float(e[:30].mean()),
                      after_dropout_max_rad=float(e[near].max()) if near.any() else None,
                      after_dropout_mean_rad=float(e[near].mean()) if near.any() else None)
    out.update(causal_ms=bc['kernel_ms'], precision=bc['precision'], mode=bc['mode'], sweeps=rec['sweeps'], converged=rec['converged'],
               ms_per_sweep=float(np.median(rec['sweep_ms'])), S_causal=rec['objective_causal'], S_joint=rec['objective'],
               max_delta=rec['max_delta'], frames_after_dropout=int(near.sum()))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sweeps', type=int, default=64)
    ap.add_argument('--cases', default='C5,C3')
    ap.add_argument('--dropout', type=int, default=12, help='frames of each of the five dropouts (0: the capture as it is)')
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    from moshpp_b200 import lib
    if lib.load_library().mosh2_device_count() < 1:
        raise SystemExit('no CUDA device: this measurement needs an H100')
    with tempfile.TemporaryDirectory() as d:
        line = dict(gpu=gpu_info(), sweeps_cap=a.sweeps, dropout=a.dropout, cases={n: run(n, a.sweeps, a.dropout, d) for n in a.cases.split(',')})
    s = json.dumps(line)
    print(s, flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(s + '\n')


if __name__ == '__main__':
    main()
