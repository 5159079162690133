"""Reporting tool (GPU): the BASELINE.json configurations C1..C4 at full size through the drop-in callable
(chmosh.mosh_stageii, default fast mode: verified time-parallel schedule), device time = sum of the launches of the call.
    python tools/gpu_configs2.py > configs.jsonl"""
import json, os, sys, tempfile, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from moshpp_b200 import chmosh, synth

d = tempfile.mkdtemp(prefix='mosh_cfg_')
for name, variants in (('C1', [{}]), ('C2', [{}]), ('C3', [{}]), ('C4', [dict(hand_side='left'), dict(hand_side='right', seq_idx=1)])):
    frames = kernel = wall = 0.0
    info = []
    for kw in variants:
        case = synth.make_case(d, name, **kw)
        best = None
        for rep in range(3):
            t0 = time.perf_counter()
            out = chmosh.mosh_stageii(case['mocap_fname'], case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])
            w = time.perf_counter() - t0
            b = out['stageii_debug_details']['b200']
            if best is None or b['kernel_ms'] < best[0]:
                best = (b['kernel_ms'], w, b)
        frames += len(out['fullpose'])
        kernel += best[0]; wall += best[1]
        b = best[2]
        info.append(dict(precision=b['precision'], chunk_len=b['chunk_len'], chunks=b['chunks'], warmup=[b['chunk_warmup'], b['warmup_full']],
                         boundary={k: b['boundary_check'][k] for k in ('rounds', 'repaired_chunks', 'chunks_over_tol_first', 'unverified_chunks')},
                         builds=b['totals']['builds'], useful_builds=b['totals']['emitted_builds']))
    print(json.dumps(dict(config=name, frames=int(frames), kernel_ms=kernel, frames_per_s_device=frames / (kernel * 1e-3),
                          call_ms=wall * 1e3, frames_per_s_call=frames / wall, detail=info)), flush=True)
