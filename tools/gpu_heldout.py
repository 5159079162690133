"""Leave-one-out held-out marker validation (``mosh_stageii(..., heldout='each')``; DESIGN.md section 12) on one GPU, on the
500-frame (BASELINE configs[1]) and the 4000-frame north-star (config 5) SMPL-H captures, each in its default mode.

Reported per capture: the main solve alone (device time of its verified launch, wall time of the call), and with leave-one-out
the device time of the fold launch (every fold in one verified launch, repairs included), its chunks and repair rounds, the wall
time of the whole call, and the overall held-out error against the main solve's own residual on the visible markers.  The
subject cache and the kernels are warmed by a first call.  Prints one JSON line with the card's name and power limit; ``--out``
also writes it.

    python tools/gpu_heldout.py --out heldout.json
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f'unknown ({e})'


def run(name, repeats):
    from bench import make_case
    from moshpp_b200 import chmosh
    case = make_case(name, 0, tag='heldout_')
    args = (case['mocap_fname'], case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])
    chmosh.mosh_stageii(*args)                                   # (warms the subject cache and the kernels)
    main_wall, main_ms, wall, rec = [], [], [], None
    for _ in range(repeats):
        t = time.perf_counter()
        out = chmosh.mosh_stageii(*args)
        main_wall.append(time.perf_counter() - t)
        main_ms.append(out['stageii_debug_details']['b200']['kernel_ms'])
        t = time.perf_counter()
        out = chmosh.mosh_stageii(*args, heldout='each')
        wall.append(time.perf_counter() - t)
        r = out['stageii_debug_details']['b200']['heldout']
        rec = rec or dict(fold_ms=[], chunks=r['chunks'], repair_rounds=[])
        rec['fold_ms'].append(r['kernel_ms'])
        rec['repair_rounds'].append(r['repair_rounds'])
    med = lambda v: float(sorted(v)[len(v) // 2])
    return dict(frames=int(len(case['obs'])), folds=len(r['folds']), fold_frames=len(r['folds']) * int(len(case['obs'])),
                precision=r['precision'], chunk_len=r['chunk_len'], main_kernel_ms=med(main_ms), main_wall_s=med(main_wall),
                fold_kernel_ms=med(rec['fold_ms']), fold_chunks=rec['chunks'], fold_repair_rounds=rec['repair_rounds'],
                heldout_call_wall_s=med(wall), heldout_overall=r['overall'], visible_overall=r['visible']['overall'],
                device_errors=r['device_errors'], repeats=repeats)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--cases', default='C2,C5')
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    from moshpp_b200 import lib
    if lib.load_library().mosh2_device_count() < 1:
        raise SystemExit('no CUDA device: this measurement needs an H100')
    line = dict(gpu=gpu_info(), cases={n: run(n, a.repeats) for n in a.cases.split(',')})
    s = json.dumps(line)
    print(s, flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(s + '\n')


if __name__ == '__main__':
    main()
