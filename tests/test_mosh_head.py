"""The head (moshpp_b200.mosh_head) end to end on a small synthetic subject of three captures: the product's Stage I on the
host build of the device source, the float64 oracle as Stage II, both injected through run_moshpp_once / run_moshpp_subject.
Pickles at the derived paths, caches on the second run, the refused surface model, the head's Stage-I keys, the Stage-II merge
and its AMASS npz, and the missing-layout error."""
import functools
import json
import os
import pickle
import shutil

import numpy as np
import pytest

from conftest import EmuStageIBackend, run_oracle
from moshpp_b200 import amass_io, mosh_head, stagei, synth
from oracle import stageii as oracle_stageii


@pytest.fixture(scope='module')
def subject(tmp_path_factory):
    root = str(tmp_path_factory.mktemp('head'))
    model_dir = os.path.join(root, 'models')
    session = os.path.join(root, 'mocap', 'Synth DS', 'subject 01')
    os.makedirs(session)
    caps, case = [], None
    for k, F in enumerate((10, 8, 12)):
        c = synth.make_case(model_dir, 'C2', frames=F, n_verts=1500, seq_idx=k)
        dst = os.path.join(session, f'take_{k:02d}.npz')
        shutil.move(c['mocap_fname'], dst)
        caps.append(dst)
        case = case or c
    with open(os.path.join(session, 'settings.json'), 'w') as f:
        json.dump({'gender': 'male'}, f)
    work = os.path.join(root, 'work')
    cfg = {'mocap.fname': caps[0], 'dirs.work_base_dir': work, 'dirs.support_base_dir': os.path.join(root, 'support'),
           'surface_model.type': 'smplh', 'surface_model.fname': case['cfg'].surface_model.fname,
           'moshpp.pose_body_prior_fname': case['cfg'].moshpp.pose_body_prior_fname,
           'moshpp.pose_hand_prior_fname': case['cfg'].moshpp.pose_hand_prior_fname, 'moshpp.optimize_fingers': True,
           'moshpp.stagei_frame_picker.num_frames': 4, 'moshpp.stagei_frame_picker.least_avail_markers': 0.8,
           'opt_settings.maxiter': 4,
           'moshpp.head_marker_corr_fname': None}      # (the yaml's default names a file; this Stage I has no head-marker prior)
    return dict(root=root, caps=caps, cfg=cfg, work=work, meta=case['marker_meta'])


def _stagei():
    return functools.partial(stagei.mosh_stagei, backend=EmuStageIBackend())


def _oracle_stageii(mocap_fname, cfg, markers_latent, latent_labels, betas, marker_meta, v_template_fname=None):
    out = oracle_stageii.mosh_stageii(mocap_fname, cfg, markers_latent, latent_labels, betas, marker_meta, v_template_fname)
    out.pop('_pose_reduced')
    out['stageii_debug_details'].pop('oracle_stats')
    return out


def _write_layout(subject):
    fname = os.path.join(subject['work'], 'SynthDS', 'SynthDS_smplh.json')
    os.makedirs(os.path.dirname(fname), exist_ok=True)
    return stagei.write_marker_layout(fname, subject['meta'])


def _equal(a, b, skip=('stageii_elapsed_time', 'stagei_elapsed_time')):
    if isinstance(a, dict):
        assert set(a) == set(b)
        for k in a:
            if k not in skip:
                _equal(a[k], b[k], skip)
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b)
        for x, y in zip(a, b):
            _equal(x, y, skip)
    elif isinstance(a, np.ndarray):
        assert a.shape == b.shape and (np.array_equal(a, b) if a.dtype != object else all(_equal(x, y, skip) is None for x, y in zip(a, b)))
    else:
        assert a == b


def test_missing_layout_is_not_created(subject):
    cfg = dict(subject['cfg'], **{'dirs.work_base_dir': os.path.join(subject['root'], 'work_nolayout')})
    with pytest.raises(FileNotFoundError, match='SynthDS_smplh.json'):
        mosh_head.run_moshpp_once(cfg, stagei_func=_stagei(), stageii_func=_oracle_stageii)


def test_run_once_writes_caches_and_reloads_them(subject):
    layout = _write_layout(subject)
    np.random.seed(0)
    mp = mosh_head.run_moshpp_once(subject['cfg'], stagei_func=_stagei(), stageii_func=_oracle_stageii)
    w = subject['work']
    assert mp.stagei_fname == f'{w}/SynthDS/subject01/male_stagei.pkl' and os.path.exists(mp.stagei_fname)
    assert mp.stageii_fname == f'{w}/SynthDS/subject01/take_00_stageii.pkl' and os.path.exists(mp.stageii_fname)
    assert os.path.exists(mp.stagei_fname.replace('.pkl', '.json'))                 # write_optimized_marker_layout
    with open(mp.stagei_fname, 'rb') as f:
        s1 = pickle.load(f)
    dbg = s1['stagei_debug_details']
    assert len(dbg['stagei_fnames']) == len(dbg['stagei_frames']) == 4 and dbg['stagei_elapsed_time'] > 0
    assert type(dbg['cfg']) is dict and type(dbg['cfg']['dirs']) is dict and dbg['cfg']['dirs']['marker_layout']['fname'] == layout
    assert all(k.startswith(os.path.dirname(subject['caps'][0])) for k in dbg['stagei_fnames'])
    relaid = stagei.load_marker_layout(mp.stagei_fname.replace('.pkl', '.json'))
    assert dict(relaid['marker_vids']) == {l: s1['markers_latent_vids'].get(l, v) for l, v in subject['meta']['marker_vids'].items()}

    with open(mp.stageii_fname, 'rb') as f:
        s2 = pickle.load(f)
    ref = _oracle_stageii(subject['caps'][0], mp.cfg, s1['markers_latent'], s1['latent_labels'], s1['betas'], s1['marker_meta'])
    want = amass_io.merge_stageii(ref, s1, mosh_head.to_container(mp.cfg), 0.0)
    _equal(s2, want)
    npz = mosh_head.MoSh.load_as_amass_npz(mp.stageii_fname)
    assert npz['gender'] == 'male' and npz['poses'].shape == s2['fullpose'].shape and npz['pose_hand'].shape[1] == 90

    def spy(**kw):
        raise AssertionError('a cached stage was run again')
    again = mosh_head.run_moshpp_once(subject['cfg'], stagei_func=spy, stageii_func=spy)
    _equal(again.stageii_data, s2, skip=())

    other = os.path.join(subject['root'], 'model_copy.pkl')
    shutil.copy(subject['cfg']['surface_model.fname'], other)
    with pytest.raises(AssertionError, match='surface_model_fname used for previous stagei'):
        mosh_head.run_moshpp_once(dict(subject['cfg'], **{'surface_model.fname': other}), stagei_func=spy, stageii_func=spy)


def test_subject_run_writes_what_per_capture_runs_write(subject):
    """run_moshpp_subject with a batch function made of per-capture oracle calls: the same pickles as run_moshpp_once of each
    capture (which reuses the Stage-I cache the first test wrote)."""
    _write_layout(subject)
    calls = []

    def batch(mocap_fnames, cfg, **kw):
        calls.append(list(mocap_fnames))
        return [_oracle_stageii(fn, cfg, **kw) for fn in mocap_fnames]
    cfg = dict(subject['cfg'], **{'dirs.work_base_dir': os.path.join(subject['root'], 'work_subject')})
    shutil.copytree(os.path.join(subject['work'], 'SynthDS'), os.path.join(cfg['dirs.work_base_dir'], 'SynthDS'))
    os.remove(os.path.join(cfg['dirs.work_base_dir'], 'SynthDS', 'subject01', 'take_00_stageii.pkl'))
    heads = mosh_head.run_moshpp_subject(cfg, stageii_batch_func=batch)
    assert calls == [subject['caps']] and [h.cfg.mocap.fname for h in heads] == subject['caps']
    for h, fn in zip(heads, subject['caps']):
        one = mosh_head.run_moshpp_once(dict(subject['cfg'], **{'mocap.fname': fn}), stageii_func=_oracle_stageii)
        assert os.path.basename(h.stageii_fname) == os.path.basename(one.stageii_fname)
        with open(h.stageii_fname, 'rb') as f:
            _equal(pickle.load(f), one.stageii_data, skip=('stageii_elapsed_time', 'work_base_dir', 'stagei_fname', 'stageii_fname',
                                                           'log_fname', 'fname'))
    again = mosh_head.run_moshpp_subject(cfg, stageii_batch_func=None, stagei_func=None)       # everything cached: no solve
    assert all(h.stageii_data is not None for h in again)


def test_head_needs_stage_i_before_stage_ii(subject):
    mp = mosh_head.MoSh(**subject['cfg'])
    with pytest.raises(ValueError, match='please run stagei first'):
        mp.mosh_stageii(_oracle_stageii)
