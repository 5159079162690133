"""The Geman-McClure data term of Stage II (``robust_data_sigma``) on one GPU: what it costs and what it recovers.

1. Cost: the north-star launch (BASELINE config 5 shape: SMPL-H, 4000 frames, default schedule: float32, planned chunks,
   verified warm-up) on one resident job per setting, sigma off and sigma = ``--sigma`` alternated for ``--repeats`` rounds
   after a warm-up of both.  Reported per setting: device time of the verified solve (CUDA events around every launch,
   repair launches included).
2. Accuracy: a 500-frame C2 capture corrupted as in tests/test_robust_data.py (a 40-frame label swap, a 30-frame ghost
   marker 0.3 m away, five isolated 0.1 m spikes), solved in the default mode with the least-squares and with the robust
   data term; worst body-pose error on the corrupted frames and on the clean frames against the float64 sequential
   least-squares solve of the clean capture.

Prints one JSON line with the card's name and power limit; ``--out`` also writes it to a file.

    python tools/gpu_robust.py --repeats 5 --out robust.json
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
sys.path.insert(0, os.path.join(ROOT, 'tests'))


def gpu_info():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f'unknown ({e})'


def cost(sigma, repeats):
    from bench import dense, make_case
    from moshpp_b200 import chmosh, lib
    case = make_case('C5', 0, tag='robust_ns_')
    pk, opts, _ = chmosh.prepare_stageii(case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])
    obs, vis = dense(case)
    F = obs.shape[0]
    w, wf = chmosh.DEFAULT_WARMUP, chmosh.DEFAULT_WARMUP_FULL
    extra = chmosh.first_chunk_extra(w, wf)
    chunk_len = chmosh.plan_chunk_len([F], chmosh.NUM_SMS, w, wf, first_extra=extra)
    tol = chmosh.BOUNDARY_TOL['fast']
    model = lib.Model(pk, device=0)
    jobs = {}
    try:
        for name, o in (('off', opts), ('on', chmosh.with_robust_sigma(opts, sigma))):
            jobs[name] = model.job(F, o, chunk_len=chunk_len, chunk_warmup=w, warmup_full=wf, precision=lib.MOSH2_F32, first_extra=extra)
            jobs[name].upload(obs, vis)
            jobs[name].sync()
        ms = {k: [] for k in jobs}
        rounds = {k: [] for k in jobs}
        for r in range(2 + repeats):
            for k, job in jobs.items():
                _, rep = chmosh.launch_verified(job, tol)
                if r >= 2:
                    ms[k].append(sum(rep['kernel_ms']))
                    rounds[k].append(rep['rounds'])
        totals = {k: job.totals() for k, job in jobs.items()}
    finally:
        for job in jobs.values():
            job.close()
        model.close()
    return dict(frames=F, chunk_len=chunk_len, device_ms={k: [round(v, 2) for v in x] for k, x in ms.items()},
                device_ms_median={k: float(np.median(x)) for k, x in ms.items()}, repair_rounds=rounds,
                totals={k: {n: int(v) for n, v in t.items()} if isinstance(t, dict) else [int(v) for v in t] for k, t in totals.items()})


def accuracy(sigma, d):
    from conftest import dense_obs
    from moshpp_b200 import chmosh, synth
    from test_robust_data import corrupt, write_capture
    case = synth.make_case(d, 'C2', frames=500)
    obs0, vis0 = dense_obs(case)
    obs, vis, bad = corrupt(obs0, vis0, swap=slice(100, 140), ghost=slice(300, 330), spikes=[30, 200, 250, 420, 470])
    args = (case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])
    ref = chmosh.mosh_stageii(case['mocap_fname'], case['cfg'], *args, precision='f64', chunk_len=0)
    fn = os.path.join(d, 'corrupted_C2.npz')
    cfg = write_capture(case, obs, vis, fn)
    bd = case['pack'].body_dof
    near = np.convolve(bad.astype(float), np.ones(16), mode='full')[:len(bad)] > 0
    out = {}
    for name, s in (('l2', None), ('robust', sigma)):
        r = chmosh.mosh_stageii(fn, copy.deepcopy(cfg), *args, robust_data_sigma=s)
        b = r['stageii_debug_details']['b200']
        assert np.array_equal(b['frame_ids'], ref['stageii_debug_details']['b200']['frame_ids'])
        e = np.abs(b['pose_reduced'][:, :bd] - ref['stageii_debug_details']['b200']['pose_reduced'][:, :bd]).max(1)
        out[name] = dict(worst_corrupted_rad=float(e[bad].max()), median_corrupted_rad=float(np.median(e[bad])),
                         worst_clean_rad=float(e[~near].max()), kernel_ms=b['kernel_ms'])
    return dict(frames=len(obs), corrupted_frames=int(bad.sum()), **out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sigma', type=float, default=0.03)
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    from moshpp_b200 import lib
    if lib.load_library().mosh2_device_count() < 1:
        raise SystemExit('no CUDA device: this measurement needs an H100')
    line = dict(gpu=gpu_info(), sigma=a.sigma, cost=cost(a.sigma, a.repeats))
    with tempfile.TemporaryDirectory() as d:
        line['accuracy'] = accuracy(a.sigma, d)
    s = json.dumps(line)
    print(s, flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(s + '\n')


if __name__ == '__main__':
    main()
