"""Generates tests/golden/long_*.npz: the SEQUENTIAL float64 oracle (the reference's schedule,
chmosh.py:584-724) on the BASELINE configurations at full size, so that the GPU parity tests can compare
the product path (f32, chunked in time, default warm-up) with it without spending GPU-box minutes on the
frame-serial numpy solve.

    python tests/golden/make_long_golden.py KEY [KEY ...]       # keys: see LONG below

Poses / translations are stored as float32 (rounding 6e-8, four orders below the tolerances they are
compared at); per-frame data SSE and frame ids as float64 / int32.  The 4000-frame sequences keep the pose (and dmpl)
rows of their first POSE_FRAMES solved frames only, so that every fixture stays below 1 MB; translations, data SSE
and frame ids cover every frame.
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from moshpp_b200 import synth  # noqa: E402
from oracle import stageii  # noqa: E402

# key -> (config, make_case kwargs).  Full-size models (n_verts=None).
LONG = {
    'C2': ('C2', dict(frames=500)),                                  # BASELINE configs[1]
    'NS': ('C5', dict(frames=4000, seq_idx=0)),                      # north-star target: 4000-frame SMPL-H sequence
    'C3': ('C3', dict(frames=640)),                                  # a window of configs[2], solved with its 4000-frame chunking
    'C3F': ('C3', dict(frames=4000)),                                # configs[2] in full: SMPL-X + DMPL, 4000 frames
    'C4L': ('C4', dict(frames=2000, hand_side='left')),              # configs[3]
    'C4R': ('C4', dict(frames=2000, hand_side='right')),
    'C5a': ('C5', dict(frames=320, seq_idx=0)),                      # configs[4] shape: several sequences, one model family
    'C5b': ('C5', dict(frames=320, seq_idx=1)),
    'C5c': ('C5', dict(frames=320, seq_idx=2)),
    'C5d': ('C5', dict(frames=320, seq_idx=3)),
    # occlusion gap straddling a chunk boundary (ADVICE r1): built by the test from C2 with frames 90..139 blanked
    'GAP': ('C2', dict(frames=240)),
    # the whole body turning about the up axis (synth.make_motion root_yaw): the root's axis-angle passes pi once (TURN), or
    # starts facing backwards and sways around pi, passing it again and again (BACK)
    'TURN': ('C2', dict(frames=600, root_yaw=(2.0, 5.0))),
    'BACK': ('C2', dict(frames=600, root_yaw=tuple(np.pi + 0.3 * np.sin(2 * np.pi * 0.4 * np.arange(600) / 120.0 - np.arcsin(1 / 6))))),
}
POSE_FRAMES = 2000      # pose / dmpl rows stored per fixture (a contiguous run from the first solved frame)


def shrink(arrs):
    """The stored subset: pose and dmpl rows of the first POSE_FRAMES solved frames."""
    return {k: (v[:POSE_FRAMES] if k in ('pose', 'dmpls') else v) for k, v in arrs.items()}


def blank_gap(case):
    """All markers missing on frames 100..129, and only 3 markers visible on 90..99 / 130..139."""
    from moshpp_b200.mocap_interface import MocapSession
    mocap = MocapSession(case['mocap_fname'], case['cfg'].mocap.unit)
    mocap.markers[100:130] = 0.0          # (0,0,0) = missing, mocap_interface.py:223-225
    keep = [mocap.labels.index(l) for l in case['latent_labels'][:3]]
    drop = [i for i in range(len(mocap.labels)) if i not in keep]
    mocap.markers[90:100][:, drop] = 0.0
    mocap.markers[130:140][:, drop] = 0.0
    return mocap


def main():
    d = tempfile.mkdtemp(prefix='mosh_long_golden_')
    for key in sys.argv[1:]:
        name, kw = LONG[key]
        case = synth.make_case(d, name, **kw)
        mocap = blank_gap(case) if key == 'GAP' else None
        out = stageii.mosh_stageii(case['mocap_fname'], case['cfg'], case['markers_latent'], case['latent_labels'],
                                   case['betas'], case['marker_meta'], mocap=mocap)
        dbg = out['stageii_debug_details']
        st = dbg['oracle_stats']
        arrs = dict(pose=out['_pose_reduced'].astype(np.float32), trans=out['trans'].astype(np.float32),
                    frame_ids=dbg['frame_ids'].astype(np.int32), err_data=dbg['stageii_errs']['data'],
                    j_evals=np.array(st['j_evals']), r_evals=np.array(st['r_evals']),
                    obs_checksum=np.array([np.nansum(case['obs']), case['vis'].sum()]))
        if 'dmpls' in out:
            arrs['dmpls'] = out['dmpls'].astype(np.float32)
        if key in ('C2', 'GAP'):
            arrs['markers_sim'] = np.concatenate(dbg['markers_sim']).astype(np.float32)
        np.savez_compressed(os.path.join(HERE, f'long_{key}.npz'), **shrink(arrs))
        print(key, out['fullpose'].shape, st, 'written', flush=True)


if __name__ == '__main__':
    main()
