"""Measures the BASELINE.json configurations on one H100 (development / reporting tool, not the product):
C1..C4 at full size through the C-ABI job calls, a C5 shard (4 sequences x 4000 frames on one GPU, jobs on
separate streams), and optionally the CPU oracle in reference-cost mode on the first frames of each config.

    python tools/gpu_configs.py [--cpu-frames 4] [--only C2,C5]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from moshpp_b200 import chmosh, lib, synth  # noqa: E402
from moshpp_b200.mocap_interface import MocapSession  # noqa: E402


def load(name, d, frames=None, seq_idx=0, hand_side='left'):
    case = synth.make_case(d, name, frames=frames, seq_idx=seq_idx, hand_side=hand_side)
    pk, opts, flags = chmosh.prepare_stageii(case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])
    mocap = MocapSession(case['mocap_fname'], case['cfg'].mocap.unit)
    obs, vis = mocap.frames_for_labels(case['latent_labels'], range(len(mocap)))
    return case, pk, opts, obs, vis


def run_jobs(items, reps=3, warmup=chmosh.DEFAULT_WARMUP, precision=lib.MOSH2_F32, sm_budget=chmosh.NUM_SMS):
    """items: list of (pk, opts, obs, vis).  All jobs are launched back to back on their own streams."""
    models = [lib.Model(pk) for pk, _, _, _ in items]
    jobs = []
    for mdl, (pk, opts, obs, vis) in zip(models, items):
        F = obs.shape[0]
        L = chmosh.auto_chunk_len(F, max(1, sm_budget // len(items)))
        if L >= F:
            L = 0
        j = mdl.job(F, opts, chunk_len=L, chunk_warmup=warmup, precision=precision)
        j.upload(obs, vis)
        jobs.append(j)
    for j in jobs:
        j.sync()
    walls = []
    for _ in range(reps + 1):
        t0 = time.perf_counter()
        for j in jobs:
            j.launch()
        for j in jobs:
            j.sync()
        walls.append(time.perf_counter() - t0)
    wall = min(walls[1:])
    res = [j.download() for j in jobs]
    tot = [j.totals() for j in jobs]
    out = dict(wall_ms=wall * 1e3, kernel_ms=[j.kernel_ms() for j in jobs], chunks=[j.num_chunks for j in jobs],
               builds=sum(t['builds'] for t in tot), evals=sum(t['evaluations'] for t in tot))
    for j in jobs:
        j.close()
    for m in models:
        m.close()
    return out, res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--cpu-frames', type=int, default=0)
    ap.add_argument('--only', default='C1,C2,C3,C4,C5')
    args = ap.parse_args()
    only = args.only.split(',')
    d = tempfile.mkdtemp(prefix='mosh_cfg_')
    for name in ('C1', 'C2', 'C3', 'C4'):
        if name not in only:
            continue
        if name == 'C4':
            loaded = [load('C4', d, hand_side='left'), load('C4', d, hand_side='right', seq_idx=1)]
        else:
            loaded = [load(name, d)]
        items = [(pk, opts, obs, vis) for (_, pk, opts, obs, vis) in loaded]
        F = sum(o.shape[0] for _, _, o, _ in items)
        out, res = run_jobs(items)
        pk = items[0][0]
        rms = []
        for (_, _, obs, vis), r in zip(items, res):
            dd = np.linalg.norm(r.markers_sim - obs, axis=-1)[vis]
            rms.append(float(np.sqrt((dd ** 2).mean()) * 1e3))
        line = dict(config=name, frames=F, markers=pk.n_markers, free_vars=len(pk.free_step2), sequences=len(items),
                    fps=F / (out['wall_ms'] * 1e-3), us_per_frame_iteration=out['wall_ms'] * 1e3 / max(1, out['builds']),
                    marker_rms_mm=rms, **out)
        if args.cpu_frames:
            from oracle import stageii
            case = loaded[0][0]
            nf = min(args.cpu_frames, items[0][2].shape[0])
            for mode in ('reference_cost', 'lean'):
                t0 = time.time()
                o = stageii.mosh_stageii(case['mocap_fname'], case['cfg'], case['markers_latent'], case['latent_labels'],
                                         case['betas'], case['marker_meta'], mode=mode, max_frames=nf)
                st = o['stageii_debug_details']['oracle_stats']
                line[f'cpu_{mode}_s_per_frame'] = st['elapsed'] / max(1, st['frames'])
                line[f'cpu_{mode}_frames'] = st['frames']
            line['host_cores'] = os.cpu_count()
        print(json.dumps(line), flush=True)
    if 'C5' in only:
        loaded = [load('C5', d, seq_idx=i) for i in range(4)]
        items = [(pk, opts, obs, vis) for (_, pk, opts, obs, vis) in loaded]
        F = sum(o.shape[0] for _, _, o, _ in items)
        out, res = run_jobs(items)
        print(json.dumps(dict(config='C5 shard (4 of the 32 sequences, 4000 frames each, one GPU)', frames=F,
                              fps=F / (out['wall_ms'] * 1e-3), us_per_frame_iteration=out['wall_ms'] * 1e3 / max(1, out['builds']) * sum(out['chunks']) / 1.0 if False else None,
                              solved=[int(((r.status & lib.ST_SOLVED) != 0).sum()) for r in res], **out)), flush=True)


if __name__ == '__main__':
    main()
