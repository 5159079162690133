"""A subject's captures in one launch: chmosh.mosh_stageii_batch (one pack, one batch job, one verified launch) and its range
upload of the raw marker tables (mosh2_job_upload_markers_range), against per-capture mosh_stageii, the host adapter and the
head's per-capture runs."""
import copy
import functools
import json
import os
import pickle
import shutil

import numpy as np
import pytest

from moshpp_b200 import chmosh, lib
from moshpp_b200.mocap_interface import MocapSession, rotation_xyz

pytestmark = pytest.mark.gpu


def _subject(tmp_path, frames=(40, 24, 33)):
    """Captures of one synthetic subject: consecutive pieces of one C2 motion (synth.make_subject)."""
    from moshpp_b200 import synth
    return synth.make_subject(str(tmp_path / 'subject'), 'C2', frames, n_verts=1500)


def _with_duplicate_label(src, dst):
    """A copy of a capture whose first label owns two columns (the host adapter's "last available one wins" rule)."""
    z = np.load(src)
    mk, labels = z['markers'], list(z['labels'])
    extra = mk[:, :1].copy()
    extra[::3] = np.nan
    np.savez(dst, markers=np.concatenate([mk, extra], 1), labels=np.array(labels + [labels[0]]), frame_rate=120.0)
    return dst


def _args(case):
    return (case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])


def _assert_same(a, b):
    for k in ('fullpose', 'trans', 'dmpls', 'expression'):
        assert (k in a) == (k in b)
        if k in a:
            assert np.array_equal(a[k], b[k]), k
    da, db = a['stageii_debug_details'], b['stageii_debug_details']
    assert set(da) == set(db)
    assert set(da['stageii_errs']) == set(db['stageii_errs'])
    for k in da['stageii_errs']:
        assert np.array_equal(da['stageii_errs'][k], db['stageii_errs'][k]), k
    for k in ('markers_sim', 'markers_obs'):
        assert len(da[k]) == len(db[k]) and all(np.array_equal(x, y) for x, y in zip(da[k], db[k])), k
    assert da['labels_obs'] == db['labels_obs'] and da['labels_orig'] == db['labels_orig']
    assert np.array_equal(da['markers_orig'], db['markers_orig'])
    for k in ('mocap_fname', 'mocap_frame_rate', 'mocap_time_length'):
        assert da[k] == db[k]
    ba, bb = da['b200'], db['b200']
    assert np.array_equal(ba['status'], bb['status']) and np.array_equal(ba['counters'], bb['counters'])
    assert np.array_equal(ba['frame_ids'], bb['frame_ids'])


@pytest.mark.parametrize('kind', ['device', 'host', 'mixed'])
def test_batch_equals_per_capture_sequential_f64(kind, tmp_path):
    case, fnames = _subject(tmp_path)
    if kind == 'mixed':
        fnames[1] = _with_duplicate_label(fnames[1], str(tmp_path / 'dup.npz'))
    kw = dict(precision='f64', chunk_len=0, device_adapter=kind != 'host')
    outs = chmosh.mosh_stageii_batch(fnames, *_args(case), **kw)
    assert len(outs) == len(fnames)
    adapters = [o['stageii_debug_details']['b200']['device_adapter'] for o in outs]
    assert adapters == {'device': [True] * 3, 'host': [False] * 3, 'mixed': [True, False, True]}[kind]
    batch = outs[0]['stageii_debug_details']['b200']['batch']
    assert batch['shared'] and batch['captures'] == 3 and batch['chunks'] == 3
    assert all(o['stageii_debug_details']['b200']['batch'] is batch for o in outs)
    for fn, o in zip(fnames, outs):
        one = chmosh.mosh_stageii(fn, *_args(case), **kw)
        _assert_same(o, one)


def test_range_upload_equals_host_adapter(tmp_path):
    """Captures that differ in column order, unit, rotation and frame range (start, stride), uploaded back to back into one
    batch job of one-frame chunks: the observations and visibility the kernel sees (read through linearise mode's weighted
    residual, zero where a marker is invisible) equal those of the host adapter uploaded as a whole."""
    case, fnames = _subject(tmp_path, frames=(40, 31, 52))
    labels = case['latent_labels']
    specs = []
    for k, (fn, unit, rot, start, step) in enumerate(zip(fnames, ('mm', 'm', 'mm'), (None, None, [10.0, -20.0, 30.0]), (0, 3, 1), (1, 2, 3))):
        z = np.load(fn)
        perm = np.random.default_rng(k).permutation(z['markers'].shape[1])
        mk = z['markers'][:, perm] / (1000.0 if unit == 'm' else 1.0)
        dst = str(tmp_path / f'cap{k}.npz')
        np.savez(dst, markers=mk, labels=z['labels'][perm], frame_rate=120.0)
        m = MocapSession(dst, mocap_unit=unit, mocap_rotate=rot)
        sel = range(start, len(m), step)
        cols = m.raw_columns_for_labels(labels)
        assert cols is not None
        obs, vis = m.frames_for_labels(labels, sel)
        specs.append(dict(m=m, sel=sel, cols=cols, obs=obs, vis=vis, rot=rot))
    pk, opts, _ = chmosh.prepare_stageii(*_args(case))
    counts = [len(s['sel']) for s in specs]
    model = lib.Model(pk, device=0)
    try:
        x = np.zeros((sum(counts), pk.nx))
        x[:, :3] = np.concatenate([np.nanmean(s['obs'], 1) for s in specs])
        a = model.job(counts, opts, chunk_len=1, precision=lib.MOSH2_F64)
        off = a.seq_offsets
        for k, s in enumerate(specs):
            rot = None if s['rot'] is None else rotation_xyz(s['rot'])
            a.upload_markers_range(int(off[k]), counts[k], s['m'].raw, s['cols'], s['sel'].start, s['sel'].step, s['m'].unit_per_metre, rot)
        ra = a.linearize(x, opts, 2, False)
        b = model.job(counts, opts, chunk_len=1, precision=lib.MOSH2_F64)
        b.upload(np.concatenate([s['obs'] for s in specs]), np.concatenate([s['vis'] for s in specs]))
        rb = b.linearize(x, opts, 2, False)
        a.close()
        b.close()
    finally:
        model.close()
    vis = np.concatenate([s['vis'] for s in specs])
    ra_r, rb_r = ra['r'].reshape(-1, len(labels), 3), rb['r'].reshape(-1, len(labels), 3)
    assert np.array_equal(ra_r == 0, rb_r == 0) and np.array_equal((rb_r != 0).any(-1), vis)
    rotated = slice(int(off[2]), int(off[3]))
    plain = np.ones(len(vis), dtype=bool)
    plain[rotated] = False
    assert np.array_equal(ra_r[plain], rb_r[plain]) and np.array_equal(ra['errs'][plain], rb['errs'][plain])
    # (the rotation is a float64 3x3 product on either side, not necessarily rounded alike in the last bit)
    assert np.abs(ra_r[rotated] - rb_r[rotated]).max() < 1e-9 * opts.wt_data
    assert (~vis).any() and vis.any()


def test_default_mode_batch_within_tolerance(tmp_path):
    """The default fast mode (float32, planned chunks, verified warm-up) over a batch: every capture within BASELINE.md
    section 4's per-frame tolerances of its own sequential float64 solve, and the boundary report covers the whole batch."""
    case, fnames = _subject(tmp_path, frames=(500, 320, 410))
    outs = chmosh.mosh_stageii_batch(fnames, *_args(case))
    batch = outs[0]['stageii_debug_details']['b200']['batch']
    assert batch['precision'] == 'f32' and batch['chunk_len'] > 0 and batch['chunks'] > 3
    bc = batch['boundary_check']
    assert bc['boundary_delta_first'] is not None and bc['unverified_chunks'] <= max(1, 0.05 * batch['chunks'])
    print(f"\nbatch of {len(fnames)}: {batch['chunks']} chunks of {batch['chunk_len']}, rounds {bc['rounds']}, "
          f"first delta {bc['boundary_delta_first']}, kernel {batch['kernel_ms']:.1f} ms")
    bd = min(case['pack'].body_dof, 66)
    for fn, o in zip(fnames, outs):
        ref = chmosh.mosh_stageii(fn, *_args(case), precision='f64', chunk_len=0)
        b, rb = o['stageii_debug_details']['b200'], ref['stageii_debug_details']['b200']
        assert np.array_equal(b['frame_ids'], rb['frame_ids'])
        dp = np.abs(b['pose_reduced'] - rb['pose_reduced'])
        body, dtr = dp[:, :bd].max(1), np.abs(o['trans'] - ref['trans']).max(1)
        assert (body > 1e-3).mean() <= 0.01 and (dtr > 1e-4).mean() <= 0.01, ((body > 1e-3).sum(), (dtr > 1e-4).sum())
        assert body.max() < 0.05 and dtr.max() < 2e-3


def test_subject_run_equals_per_capture_runs(tmp_path):
    """run_moshpp_subject writes the Stage-II pickles one run_moshpp_once per capture writes: float64 sequential arrays equal,
    only timing entries differ."""
    from moshpp_b200 import mosh_head, stagei
    case, fnames = _subject(tmp_path)
    session = tmp_path / 'mocap' / 'DS' / 'subj'
    session.mkdir(parents=True)
    caps = []
    for k, fn in enumerate(fnames):
        caps.append(str(session / f'take_{k}.npz'))
        shutil.copy(fn, caps[-1])
    (session / 'settings.json').write_text(json.dumps({'gender': 'male'}))
    cfg = case['cfg']
    base = {'mocap.fname': caps[0], 'dirs.support_base_dir': str(tmp_path / 'support'), 'surface_model.type': 'smplh',
            'surface_model.fname': cfg.surface_model.fname, 'moshpp.pose_body_prior_fname': cfg.moshpp.pose_body_prior_fname,
            'moshpp.pose_hand_prior_fname': cfg.moshpp.pose_hand_prior_fname, 'moshpp.optimize_fingers': True,
            'moshpp.head_marker_corr_fname': None, 'moshpp.stagei_frame_picker.num_frames': 4,
            'moshpp.stagei_frame_picker.least_avail_markers': 0.8, 'opt_settings.maxiter': 4}
    for w in ('w_once', 'w_subject'):
        layout = tmp_path / w / 'DS' / 'DS_smplh.json'
        layout.parent.mkdir(parents=True)
        stagei.write_marker_layout(str(layout), case['marker_meta'])
    np.random.seed(0)
    first = mosh_head.run_moshpp_once(dict(base, **{'dirs.work_base_dir': str(tmp_path / 'w_once')}), stagei_func=None,
                                      stageii_func=functools.partial(chmosh.mosh_stageii, precision='f64', chunk_len=0))
    os.makedirs(tmp_path / 'w_subject' / 'DS' / 'subj')
    shutil.copy(first.stagei_fname, tmp_path / 'w_subject' / 'DS' / 'subj')      # one Stage I for both
    heads = mosh_head.run_moshpp_subject(dict(base, **{'dirs.work_base_dir': str(tmp_path / 'w_subject')}),
                                         stageii_batch_func=functools.partial(chmosh.mosh_stageii_batch, precision='f64', chunk_len=0))
    for h, fn in zip(heads, caps):
        one = mosh_head.run_moshpp_once(dict(base, **{'mocap.fname': fn, 'dirs.work_base_dir': str(tmp_path / 'w_once')}),
                                        stageii_func=functools.partial(chmosh.mosh_stageii, precision='f64', chunk_len=0))
        with open(h.stageii_fname, 'rb') as f:
            got = pickle.load(f)
        want = one.stageii_data
        _assert_same(got, want)
        gd, wd = got['stageii_debug_details'], want['stageii_debug_details']
        cg, cw = copy.deepcopy(gd['cfg']), copy.deepcopy(wd['cfg'])
        for c in (cg, cw):
            c['dirs'] = {k: v for k, v in c['dirs'].items() if k in ('session_subject_subfolders', 'stagei_basename')}
        assert cg == cw
        assert set(got) == set(want) and np.array_equal(got['betas'], want['betas'])
