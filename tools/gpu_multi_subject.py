"""Many subjects: one ``mosh_stageii_batch`` call per subject against one ``mosh_stageii_subjects`` call, on one GPU.

Synthetic dataset (``synth.make_subject`` at full size, BASELINE config 2's SMPL-H model, layout and motion generator): every
subject has its own shape and latent markers, every fourth subject uses a second model file of the same family.  Two shapes:
``short`` = 16 subjects x 2 captures of 300-800 frames, ``long`` = 8 subjects x 8 captures of 1000-4000 frames.  Both ways run in
the default mode (float32, planned chunks, verified warm-up); after a warm-up of both, ``--repeats`` rounds alternate them.
Reported per round: device time (sum of the CUDA-event times of every launch, repair launches included) and wall time of the
whole call(s), plus frames per second.  Prints one JSON line per shape; ``--out`` also writes them to a file.

    python tools/gpu_multi_subject.py --repeats 3 --out multi_subject.json
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = {'short': (16, 2, 300, 800), 'long': (8, 8, 1000, 4000)}     # subjects, captures per subject, frames (min, max)


def gpu_info():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f'unknown ({e})'


def measure(name, repeats, seed, d):
    from moshpp_b200 import chmosh, synth
    n_sub, n_cap, lo, hi = SHAPES[name]
    rng = np.random.default_rng(seed)
    t = time.time()
    subjects = []
    for k in range(n_sub):
        frames = [int(f) for f in rng.integers(lo, hi + 1, n_cap)]
        case, fnames = synth.make_subject(os.path.join(d, name), 'C2', frames, seq_idx=k, model_seed=1 if k % 4 == 3 else 0)
        subjects.append(dict(cfg=case['cfg'], mocap_fnames=fnames, markers_latent=case['markers_latent'],
                             latent_labels=case['latent_labels'], betas=case['betas'], marker_meta=case['marker_meta']))
    gen_s = time.time() - t
    n = 0
    for s in subjects:
        for fn in s['mocap_fnames']:
            n += int(fn.rsplit('_', 1)[1].split('.')[0])

    def per_subject():
        t0 = time.perf_counter()
        outs = [chmosh.mosh_stageii_batch(s['mocap_fnames'], s['cfg'], s['markers_latent'], s['latent_labels'], s['betas'],
                                          s['marker_meta']) for s in subjects]
        wall = time.perf_counter() - t0
        return sum(o[0]['stageii_debug_details']['b200']['batch']['kernel_ms'] for o in outs), wall * 1e3, outs

    def one_call():
        t0 = time.perf_counter()
        outs = chmosh.mosh_stageii_subjects(subjects)
        wall = time.perf_counter() - t0
        batches = {id(b): b for b in (c['stageii_debug_details']['b200']['batch'] for o in outs for c in o)}
        return sum(b['kernel_ms'] for b in batches.values()), wall * 1e3, outs

    _, _, o1 = per_subject()
    _, _, o2 = one_call()
    rounds = []
    for _ in range(repeats):
        pk, pw, _ = per_subject()
        sk, sw, _ = one_call()
        rounds.append(dict(per_subject_kernel_ms=pk, per_subject_wall_ms=pw, subjects_kernel_ms=sk, subjects_wall_ms=sw))
    dev = max(float(np.abs(x['trans'] - y['trans']).max()) for a, b in zip(o1, o2) for x, y in zip(a, b))
    bt = o2[0][0]['stageii_debug_details']['b200']['batch']
    med = {k: float(np.median([r[k] for r in rounds])) for k in rounds[0]}
    return dict(shape=name, gpu=gpu_info(), subjects=n_sub, captures_per_subject=n_cap, frames_range=[lo, hi], total_frames=n,
                generate_s=gen_s, rounds=rounds, median=med,
                per_subject_frames_per_s_device=n / med['per_subject_kernel_ms'] * 1e3,
                subjects_frames_per_s_device=n / med['subjects_kernel_ms'] * 1e3,
                per_subject_frames_per_s_wall=n / med['per_subject_wall_ms'] * 1e3,
                subjects_frames_per_s_wall=n / med['subjects_wall_ms'] * 1e3,
                launches=bt['launches'], chunks=bt['chunks'], chunk_len=bt['chunk_len'], repair_rounds=bt['boundary_check']['rounds'],
                unverified_chunks=bt['boundary_check']['unverified_chunks'],
                max_trans_difference_subjects_vs_per_subject_m=dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--shapes', default='short,long')
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    from moshpp_b200 import lib
    if lib.load_library().mosh2_device_count() < 1:
        raise SystemExit('no CUDA device: this measurement needs an H100')
    lines = []
    with tempfile.TemporaryDirectory() as d:
        for name in a.shapes.split(','):
            line = json.dumps(measure(name, a.repeats, a.seed, d))
            print(line, flush=True)
            lines.append(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write('\n'.join(lines) + '\n')


if __name__ == '__main__':
    main()
