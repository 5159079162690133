"""Stage-I frame picker (moshpp_b200.frame_picker) against the picks of the reference's own, unmodified
frame_picker.py:43-213, recorded in tests/golden/ref_frame_picker.npz by make_frame_picker_vectors.py: random (several
seeds, the threshold-lowering recursion that drops exclude_markers, the > 100 stop, subjects and marker lists), random_strict
(reseeding, unreadable captures, availability over all columns, the two errors) and manual."""
import json
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'golden'))

from make_frame_picker_vectors import run_case, strip_dir  # noqa: E402

GOLDEN = os.path.join(HERE, 'golden', 'ref_frame_picker.npz')


@pytest.fixture(scope='module')
def golden(tmp_path_factory):
    z = np.load(GOLDEN)
    d = str(tmp_path_factory.mktemp('captures'))
    for i in range(int(z['n_captures'])):
        p = os.path.join(d, str(z[f'cap{i}_path']))
        os.makedirs(os.path.dirname(p), exist_ok=True)
        np.savez(p, markers=z[f'cap{i}_markers'], labels=z[f'cap{i}_labels'], frame_rate=120.0)
    cases = json.loads(str(z['cases']))
    for c in cases:
        c['fnames'] = [f.replace('<dir>', d) for f in c['fnames']]
    return d, cases, json.loads(str(z['results']))


def test_golden_covers_every_path(golden):
    _, cases, results = golden
    modes = {(c['mode'], r.get('error', 'picks')) for c, r in zip(cases, results)}
    assert modes >= {('random', 'picks'), ('random', 'ValueError'), ('random_strict', 'picks'), ('random_strict', 'ValueError'),
                     ('random_strict', 'AssertionError'), ('manual', 'picks'), ('manual', 'AssertionError')}


@pytest.mark.parametrize('i', range(30))
def test_picks_equal_the_reference_picker(golden, i):
    from moshpp_b200 import frame_picker
    d, cases, results = golden
    got = strip_dir(run_case(frame_picker, cases[i]), d)
    want = results[i]
    if 'error' in want:
        assert got == want
        return
    assert got['keys'] == want['keys']
    assert len(got['frames']) == len(want['frames'])
    for a, b in zip(got['frames'], want['frames']):
        assert list(a.keys()) == list(b.keys())
        assert all(a[k] == b[k] for k in a)          # bit for bit


def test_random_lowers_the_threshold_and_drops_exclude_markers(golden, monkeypatch):
    """Labels with a '*' inside never count as available, so no frame of that capture reaches 100 %: the threshold goes
    down in 0.01 steps, and from the first lowering on the excluded labels are back (frame_picker.py:142-145)."""
    from moshpp_b200 import frame_picker
    d, cases, _ = golden
    c = next(c for c in cases if c['mode'] == 'random' and 'X*1' in (c['kw'].get('exclude_markers') or ()))
    calls = []
    orig = frame_picker.load_marker_sessions_random

    def spy(*a, **kw):
        calls.append((kw.get('least_avail_markers'), kw.get('exclude_markers')))
        return orig(*a, **kw)
    monkeypatch.setattr(frame_picker, 'load_marker_sessions_random', spy)
    np.random.seed(c['pre'])
    frames, keys = spy(list(c['fnames']), mocap_unit='mm', **c['kw'])
    assert len(calls) > 2 and calls[0][1] and all(e is None for _, e in calls[1:])
    assert len(frames) == 6 and all('X*1' in f and 'LFHD' in f for f in frames)
