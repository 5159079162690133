"""A subject's captures per capture (one ``mosh_stageii`` call each) against one ``mosh_stageii_batch`` call, on one GPU.

Synthetic subject: ``--captures`` SMPL-H captures of 1000-4000 frames of one subject (``synth.make_subject``: BASELINE config
2's model, layout and motion generator at full size; one motion cut into consecutive captures).  Both ways run in the
default mode (float32, planned chunks, verified warm-up) with the subject cache warm; after a warm-up of both, ``--repeats`` rounds alternate them.
Reported per round: device time (sum of the CUDA-event times of every launch, repair launches included) and wall time of the
whole call(s), plus the frames per second of both.  Prints one JSON line; ``--out`` also writes it to a file.

    python tools/gpu_subject_batch.py --captures 8 --repeats 5 --out subject_batch.json
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


def gpu_info():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f'unknown ({e})'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--captures', type=int, default=8)
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    from moshpp_b200 import chmosh, lib, synth
    if lib.load_library().mosh2_device_count() < 1:
        raise SystemExit('no CUDA device: this measurement needs an H100')
    rng = np.random.default_rng(a.seed)
    frames = [int(f) for f in rng.integers(1000, 4001, a.captures)]
    with tempfile.TemporaryDirectory() as d:
        t = time.time()
        c0, fnames = synth.make_subject(d, 'C2', frames)
        gen_s = time.time() - t
        args = (c0['cfg'], c0['markers_latent'], c0['latent_labels'], c0['betas'], c0['marker_meta'])

        def per_capture():
            t0 = time.perf_counter()
            outs = [chmosh.mosh_stageii(fn, *args) for fn in fnames]
            wall = time.perf_counter() - t0
            return sum(o['stageii_debug_details']['b200']['kernel_ms'] for o in outs), wall * 1e3, outs

        def batch():
            t0 = time.perf_counter()
            outs = chmosh.mosh_stageii_batch(fnames, *args)
            wall = time.perf_counter() - t0
            return outs[0]['stageii_debug_details']['b200']['batch']['kernel_ms'], wall * 1e3, outs

        _, _, o1 = per_capture()
        _, _, o2 = batch()
        rounds = []
        for _ in range(a.repeats):
            pk, pw, _ = per_capture()
            bk, bw, _ = batch()
            rounds.append(dict(per_capture_kernel_ms=pk, per_capture_wall_ms=pw, batch_kernel_ms=bk, batch_wall_ms=bw))
        dev = max(float(np.abs(x['trans'] - y['trans']).max()) for x, y in zip(o1, o2))
        unverified = sum(o['stageii_debug_details']['b200']['boundary_check']['unverified_chunks'] for o in o1)
        bt = o2[0]['stageii_debug_details']['b200']['batch']
    n = int(sum(frames))
    med = {k: float(np.median([r[k] for r in rounds])) for k in rounds[0]}
    res = dict(gpu=gpu_info(), captures=a.captures, frames=frames, total_frames=n, generate_s=gen_s, rounds=rounds, median=med,
               per_capture_frames_per_s_device=n / med['per_capture_kernel_ms'] * 1e3,
               batch_frames_per_s_device=n / med['batch_kernel_ms'] * 1e3,
               per_capture_frames_per_s_wall=n / med['per_capture_wall_ms'] * 1e3,
               batch_frames_per_s_wall=n / med['batch_wall_ms'] * 1e3,
               batch_chunks=bt['chunks'], batch_chunk_len=bt['chunk_len'], batch_repair_rounds=bt['boundary_check']['rounds'],
               batch_unverified_chunks=bt['boundary_check']['unverified_chunks'], per_capture_unverified_chunks=unverified,
               max_trans_difference_batch_vs_per_capture_m=dev)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
