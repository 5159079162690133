"""Generates tests/golden/ref_frame_picker.npz: the Stage-I frames the UNMODIFIED reference frame picker
(moshpp.frame_picker, frame_picker.py:43-213) picks from synthetic captures.

The reference picker imports ``moshpp.tools.mocap_interface`` for ``MocapSession``, whose module needs ezc3d, psbody and
body_visualizer (absent here).  A stand-in module exposing moshpp_b200's ``MocapSession`` is put into ``sys.modules`` first
(as tests/golden/ref_shim stands in for chumpy), so what is pinned is the picker's own logic: its ``np.random`` calls, keys,
thresholds and error paths.  Every case records the seed the global legacy RNG was set to before the call, the arguments,
and the picks (keys with the capture directory replaced by ``<dir>``, and the frames' ``{label: xyz}`` dictionaries) or the
exception type.

    python tests/golden/make_frame_picker_vectors.py <moshpp source directory, the one that holds the moshpp package>
"""
import json
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)


def make_captures(rng):
    """(relative path, markers [F, L, 3] mm with NaN / zero gaps, labels) of a few synthetic captures."""
    body = ['LFHD', 'RFHD', 'LBHD', 'RBHD', 'C7', 'T10', 'CLAV', 'STRN', 'LSHO', 'RSHO', 'LELB', 'RELB', 'LWRA', 'RWRA',
            'LASI', 'RASI', 'LKNE', 'RKNE', 'LANK', 'RANK']
    caps = []

    def cap(rel, F, labels, p_gap, zeros=True):
        mk = rng.normal(0.0, 300.0, (F, len(labels), 3)) + 1000.0
        gap = rng.random((F, len(labels))) < p_gap
        mk[gap] = np.nan
        if zeros:
            z = rng.random((F, len(labels))) < p_gap / 3
            mk[z] = 0.0
        caps.append((rel, mk, list(labels)))

    cap('subj_A/walk_01.npz', 37, body + ['*12', 'EXTRA'], 0.02)
    cap('subj_A/run_02.npz', 23, body[:16] + ['L FHD2'], 0.08)                     # a blank inside a label
    cap('subj_A/jump_03.npz', 51, body, 0.0, zeros=False)                           # complete frames
    cap('subj_A/sparse_04.npz', 19, body, 0.35)                                     # many gaps: too few frames for random_strict
    cap('subj_M/duo_01.npz', 29, [f'alice:{l}' for l in body] + [f'bob:{l}' for l in body], 0.05)   # two subjects
    cap('subj_A/starred_05.npz', 21, body + ['X*1', 'X*2'], 0.0, zeros=False)       # labels with a '*' inside: < 100 %
    cap('subj_S/stars_01.npz', 15, ['LFHD*', 'RFHD*', 'C7*'], 0.1)                  # no label counts for `random`
    return caps


def cases_for(paths):
    A = [paths['subj_A/walk_01.npz'], paths['subj_A/run_02.npz'], paths['subj_A/jump_03.npz']]
    sparse = [paths['subj_A/sparse_04.npz']]
    duo = [paths['subj_M/duo_01.npz']]
    stars = [paths['subj_S/stars_01.npz']]
    starred = [paths['subj_A/starred_05.npz']]
    out = []
    for pre in (0, 1, 2):
        for seed in (100, 7, None):
            out.append(dict(mode='random', pre=pre, fnames=A, kw=dict(num_frames=12, seed=seed, least_avail_markers=1.0)))
    out += [
        dict(mode='random', pre=3, fnames=A, kw=dict(num_frames=5, seed=3, least_avail_markers=0.5)),
        dict(mode='random', pre=4, fnames=sparse + A, kw=dict(num_frames=8, seed=11, least_avail_markers=1.0)),
        dict(mode='random', pre=5, fnames=sparse, kw=dict(num_frames=10, seed=5, least_avail_markers=1.0,
                                                          exclude_markers=['LFHD', 'RFHD', 'LBHD'])),
        dict(mode='random', pre=5, fnames=starred + A, kw=dict(num_frames=20, seed=5, least_avail_markers=1.0)),   # lowered
        dict(mode='random', pre=6, fnames=starred, kw=dict(num_frames=6, seed=5, least_avail_markers=1.0,
                                                           exclude_markers=['X*1', 'LFHD'])),      # lowered, then X*1 is back
        dict(mode='random', pre=6, fnames=duo, kw=dict(num_frames=6, seed=100, least_avail_markers=1.0, only_subjects=['bob'])),
        dict(mode='random', pre=7, fnames=A * 4, kw=dict(num_frames=12, seed=100, least_avail_markers=0.9)),  # the > 100 stop
        dict(mode='random', pre=8, fnames=A, kw=dict(num_frames=4, seed=1, least_avail_markers=1.0, only_markers=['C7', 'T10', 'CLAV'])),
        dict(mode='random', pre=9, fnames=stars, kw=dict(num_frames=3, seed=1, least_avail_markers=0.1)),       # ValueError
    ]
    for seed in (100, 7, 12345):
        out.append(dict(mode='random_strict', pre=0, fnames=A, kw=dict(num_frames=12, seed=seed, least_avail_markers=1.0)))
    out += [
        dict(mode='random_strict', pre=0, fnames=A + sparse, kw=dict(num_frames=12, seed=100, least_avail_markers=0.8)),
        dict(mode='random_strict', pre=0, fnames=A, kw=dict(num_frames=6, seed=100, least_avail_markers=0.9,
                                                           exclude_markers=['C7', 'T10'])),
        dict(mode='random_strict', pre=0, fnames=duo + A, kw=dict(num_frames=6, seed=100, least_avail_markers=0.9,
                                                                 only_subjects=['alice'])),     # A: no subject 'alice'
        dict(mode='random_strict', pre=0, fnames=A * 3, kw=dict(num_frames=12, seed=9, least_avail_markers=0.5)),   # > 100
        dict(mode='random_strict', pre=0, fnames=sparse, kw=dict(num_frames=12, seed=100, least_avail_markers=1.0)),  # ValueError
        dict(mode='random_strict', pre=0, fnames=A, kw=dict(num_frames=4, seed=100, least_avail_markers=0.05)),   # AssertionError
        dict(mode='manual', pre=0, fnames=[A[0] + '_3', A[1] + '_0', A[0] + '_36', duo[0] + '_7'], kw=dict()),
        dict(mode='manual', pre=0, fnames=[duo[0] + '_2', duo[0] + '_28'], kw=dict(only_subjects=['bob'], exclude_markers=['C7'])),
        dict(mode='manual', pre=0, fnames=[A[0] + '_1', os.path.join(os.path.dirname(A[0]), 'missing.npz') + '_4'], kw=dict()),
    ]
    return out


def run_case(picker, c, unit='mm'):
    """The picker's result as plain data: {'keys': [...], 'frames': [{label: [x, y, z]}]} or {'error': type name}."""
    fn = {'random': picker.load_marker_sessions_random, 'random_strict': picker.load_marker_sessions_random_strict,
          'manual': picker.load_marker_sessions_manual}[c['mode']]
    np.random.seed(c['pre'])
    try:
        frames, keys = fn(list(c['fnames']), mocap_unit=unit, **c['kw'])
    except (ValueError, AssertionError) as e:
        return {'error': type(e).__name__}
    return {'keys': [str(k) for k in keys], 'frames': [{k: np.asarray(v).tolist() for k, v in d.items()} for d in frames]}


def write_captures(d, caps):
    paths = {}
    for rel, mk, labels in caps:
        p = os.path.join(d, rel)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        np.savez(p, markers=mk, labels=np.array(labels), frame_rate=120.0)
        paths[rel] = p
    return paths


def strip_dir(res, d):
    if 'keys' in res:
        res = dict(res, keys=[k.replace(d, '<dir>') for k in res['keys']])
    return res


def main(ref_src: str):
    from moshpp_b200 import mocap_interface
    stand_in = types.ModuleType('moshpp.tools.mocap_interface')
    stand_in.MocapSession = mocap_interface.MocapSession
    sys.path.insert(0, ref_src)
    import moshpp.tools
    sys.modules['moshpp.tools.mocap_interface'] = stand_in
    moshpp.tools.mocap_interface = stand_in
    from moshpp import frame_picker as ref_picker                 # the reference, unmodified

    caps = make_captures(np.random.default_rng(20261016))
    with tempfile.TemporaryDirectory() as d:
        paths = write_captures(d, caps)
        cases = cases_for(paths)
        results = [strip_dir(run_case(ref_picker, c), d) for c in cases]
        for c in cases:
            c['fnames'] = [f.replace(d, '<dir>') for f in c['fnames']]
    arrays = {}
    for i, (rel, mk, labels) in enumerate(caps):
        arrays[f'cap{i}_markers'] = mk
        arrays[f'cap{i}_labels'] = np.array(labels)
        arrays[f'cap{i}_path'] = np.array(rel)
    arrays['n_captures'] = np.array(len(caps))
    arrays['cases'] = np.array(json.dumps(cases))
    arrays['results'] = np.array(json.dumps(results))
    np.savez_compressed(os.path.join(HERE, 'ref_frame_picker.npz'), **arrays)
    kinds = {}
    for r in results:
        kinds[r.get('error', 'picks')] = kinds.get(r.get('error', 'picks'), 0) + 1
    print('ref_frame_picker.npz:', len(cases), 'cases', kinds)


if __name__ == '__main__':
    if len(sys.argv) != 2 or not os.path.isfile(os.path.join(sys.argv[1], 'moshpp', 'frame_picker.py')):
        raise SystemExit('usage: make_frame_picker_vectors.py <directory that holds the moshpp package of the reference>')
    main(sys.argv[1])
