"""Development tool (GPU): Stage I at BASELINE size -- twelve frames of the 4000-frame SMPL-H sequence, 53 markers, 16 shape
coefficients -- through moshpp_b200.stagei.mosh_stagei; with --oracle also the float64 oracle on the host cores (parity + time).
--face80: SMPL-X with face markers at the reference's size (16 free betas, 80 expressions), the shape and every picked frame's
jaw and expressions fitted together (face_with_free_shape).
--reference-options: with the head-marker correlation prior (a synthetic K x H file over the LFHD / RFHD / LBHD / RBHD
markers) and the extra initial rigid adjustment, both through reference_options=True.
--robust-data-sigma S: the Geman-McClure data term at sigma = S metres (robust_data_sigma).
With --oracle the float64 oracle runs with the same keywords as the library.
Usage: python tools/gpu_stagei.py [--oracle] [--frames 12] [--face80] [--reference-options] [--robust-data-sigma S]"""
import argparse
import copy
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from moshpp_b200 import stagei, synth  # noqa: E402
from moshpp_b200.mocap_interface import MocapSession  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--oracle', action='store_true')
    ap.add_argument('--frames', type=int, default=12)
    ap.add_argument('--config', default='C5')
    ap.add_argument('--face80', action='store_true')
    ap.add_argument('--reference-options', action='store_true')
    ap.add_argument('--robust-data-sigma', type=float, default=None)
    a = ap.parse_args()
    d = tempfile.mkdtemp(prefix='mosh_stagei_')
    if a.face80:
        a.config = 'CF'
    case = synth.make_case(d, a.config, frames=480, **(synth.REFERENCE_FACE if a.face80 else {}))
    cfg = copy.deepcopy(case['cfg'])
    cfg.moshpp.optimize_betas = True
    kw = dict(face_with_free_shape=True) if a.face80 else {}
    if a.reference_options:
        head = [l for l in ('LFHD', 'RFHD', 'LBHD', 'RBHD') if l in case['marker_meta']['marker_vids']]
        rng = np.random.default_rng(0)
        corr = np.vstack([np.eye(len(head)) + rng.normal(0, 0.2, (len(head), len(head))), rng.normal(0, 0.5, (2, len(head)))])
        cfg.moshpp.head_marker_corr_fname = os.path.join(d, 'ssm_head_marker_corr.npz')
        np.savez(cfg.moshpp.head_marker_corr_fname, mrk_labels=np.asarray(head), corr=corr)
        cfg.opt_settings.extra_initial_rigid_adjustment = True
        kw['reference_options'] = True
    if a.robust_data_sigma is not None:
        kw['robust_data_sigma'] = a.robust_data_sigma
    mocap = MocapSession(case['mocap_fname'], cfg.mocap.unit)
    frames = mocap.markers_asdict()
    pick = np.linspace(0, len(frames) - 1, a.frames).astype(int)
    frames = [frames[i] for i in pick]
    stagei.DeviceBackend()                  # (loads the library outside the timed call)
    t0 = time.perf_counter()
    out = stagei.mosh_stagei(frames, cfg, marker_meta=case['marker_meta'], **kw)
    dt = time.perf_counter() - t0
    st = out['stagei_debug_details']['b200']
    nb = cfg.surface_model.num_betas
    line = {'workload': f'Stage I: {a.frames} frames, {len(out["latent_labels"])} markers, {nb} betas, model {cfg.surface_model.type}',
            'seconds': dt, 'stats': st, 'errs': out['stagei_debug_details']['stagei_errs'],
            'betas_err_vs_truth': float(np.abs(out['betas'][:nb] - case['betas'][:nb]).max()),
            'latent_err_vs_truth_mm': float(1e3 * np.abs(out['markers_latent'] - case['markers_latent']).max())}
    if a.face80:
        line['workload'] += ', face: jaw + 80 expressions per frame, shape free'
    if a.reference_options:
        line['workload'] += ', head-marker correlation prior + extra initial rigid adjustment'
    if a.robust_data_sigma is not None:
        line['workload'] += f', Geman-McClure data term at sigma = {a.robust_data_sigma} m'
    if a.oracle:
        from oracle import stagei as ostagei
        t0 = time.perf_counter()
        ref = ostagei.mosh_stagei(frames, cfg, marker_meta=case['marker_meta'], **kw)
        line['oracle_seconds'] = time.perf_counter() - t0
        line['oracle_stats'] = ref['stagei_debug_details']['oracle_stats']
        line['d_betas'] = float(np.abs(out['betas'] - ref['betas']).max())
        line['d_latent'] = float(np.abs(out['markers_latent'] - ref['markers_latent']).max())
        line['d_pose'] = float(max(np.abs(p - q).max() for p, q in zip(out['stagei_debug_details']['opt_models_pose'],
                                                                        ref['stagei_debug_details']['opt_models_pose'])))
        if 'opt_models_expression' in ref['stagei_debug_details']:
            line['d_expr'] = float(max(np.abs(p - q).max() for p, q in zip(out['stagei_debug_details']['opt_models_expression'],
                                                                            ref['stagei_debug_details']['opt_models_expression'])))
    print(json.dumps(line))


if __name__ == '__main__':
    main()
