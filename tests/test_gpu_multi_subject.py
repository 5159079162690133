"""Several subjects in one launch on the H100: the multi-model job (mosh2_job_create_multi) against separate batch jobs of each
subject, chmosh.mosh_stageii_subjects against the float64 oracle, the refusal of models of another kernel shape, and the
dataset head mosh_head.run_moshpp_jobs against run_moshpp_once of every job."""
import copy
import functools
import json
import os
import pickle
import shutil

import numpy as np
import pytest

from moshpp_b200 import chmosh, lib, synth
from moshpp_b200.mocap_interface import MocapSession

pytestmark = pytest.mark.gpu


def _subjects(root, frames, n_verts=1500):
    """Three SMPL-H subjects of other shapes and latent markers; the third on a second model file."""
    out = []
    for k, fr in enumerate(frames):
        case, fnames = synth.make_subject(root, 'C2', fr, n_verts=n_verts, seq_idx=k, model_seed=1 if k == 2 else 0)
        out.append(dict(case=case, fnames=fnames))
    return out


def _stagei_outputs(case):
    return {k: case[k] for k in ('markers_latent', 'latent_labels', 'betas', 'marker_meta')}


@pytest.mark.parametrize('precision', ['f32', 'f64'])
def test_multi_launch_equals_separate_batches(tmp_path, precision):
    """One multi-model launch with verification and repair against one batch launch per subject, same explicit schedule: the
    rows of every capture, bit for bit, and the same boundary repairs."""
    subs = _subjects(str(tmp_path), [(150, 90), (120,), (80, 130)])
    prec = {'f32': lib.MOSH2_F32, 'f64': lib.MOSH2_F64}[precision]
    sched = dict(chunk_len=24, chunk_warmup=16, warmup_full=12, first_extra=chmosh.first_chunk_extra(16, 12), precision=prec)
    tol = chmosh.BOUNDARY_TOL['fast']
    models, opts, data = [], None, []
    try:
        for s in subs:
            pk, opts, _ = chmosh.prepare_stageii(s['case']['cfg'], **_stagei_outputs(s['case']))
            models.append(lib.Model(pk, device=0))
            ov = []
            for fn in s['fnames']:
                m = MocapSession(fn, s['case']['cfg'].mocap.unit)
                ov.append(m.frames_for_labels(s['case']['latent_labels'], range(len(m))))
            data.append(ov)
        order = [(0, 0), (1, 0), (2, 0), (0, 1), (2, 1)]
        job = lib.multi_job(models, [k for k, _ in order], [len(data[k][c][0]) for k, c in order], opts, **sched)
        job.upload(np.concatenate([data[k][c][0] for k, c in order]), np.concatenate([data[k][c][1] for k, c in order]))
        bad, report = chmosh.launch_verified(job, tol)
        res = chmosh.download_verified(job, bad, report)
        offs = job.seq_offsets
        assert report['rounds'] > 0 or report['chunks_over_tol_first'] == 0
        repaired = 0
        for k, (model, ov) in enumerate(zip(models, data)):
            one = model.job([len(o) for o, _ in ov], opts, **sched)
            one.upload(np.concatenate([o for o, _ in ov]), np.concatenate([v for _, v in ov]))
            b1, r1 = chmosh.launch_verified(one, tol)
            res1 = chmosh.download_verified(one, b1, r1)
            repaired += sum(r1['repaired_chunks'])
            own = one.seq_offsets
            for q, (kk, c) in enumerate(order):
                if kk != k:
                    continue
                a, b = slice(offs[q], offs[q + 1]), slice(own[c], own[c + 1])
                for name in ('fullpose', 'pose', 'trans', 'markers_sim', 'errs', 'status', 'counters'):
                    assert np.array_equal(getattr(res, name)[a], getattr(res1, name)[b]), (precision, q, name)
            one.close()
        assert sum(report['repaired_chunks']) == repaired
        print(f"\n{precision}: {job.num_chunks} chunks, {report['rounds']} repair rounds, {repaired} chunks repaired")
        job.close()
    finally:
        for m in models:
            m.close()


def test_subjects_sequential_f64_equal_oracle(tmp_path):
    """Three small SMPL-H subjects (one on a second model file) in one launch of mosh_stageii_subjects, float64 and sequential:
    every capture within BASELINE.md section 4's small-case gates of the float64 oracle."""
    from oracle import stageii as oracle_stageii
    subs = _subjects(str(tmp_path), [(10, 8), (12,), (9, 7)])
    outs = chmosh.mosh_stageii_subjects([dict(cfg=s['case']['cfg'], mocap_fnames=s['fnames'], **_stagei_outputs(s['case'])) for s in subs],
                                        precision='f64', chunk_len=0)
    assert [len(o) for o in outs] == [2, 1, 2]
    batch = outs[0][0]['stageii_debug_details']['b200']['batch']
    assert batch['launches'] == 1 and batch['subjects'] == 3 and batch['captures'] == 5 and batch['chunks'] == 5
    for s, so in zip(subs, outs):
        c = s['case']
        for fn, o in zip(s['fnames'], so):
            ref = oracle_stageii.mosh_stageii(fn, c['cfg'], c['markers_latent'], c['latent_labels'], c['betas'], c['marker_meta'])
            dbg, rdbg = o['stageii_debug_details'], ref['stageii_debug_details']
            assert np.array_equal(dbg['b200']['frame_ids'], rdbg['frame_ids'])
            assert np.abs(dbg['b200']['pose_reduced'] - ref['_pose_reduced']).max() < 1e-8
            assert np.abs(o['fullpose'] - ref['fullpose']).max() < 1e-8
            assert np.abs(o['trans'] - ref['trans']).max() < 1e-9
            for k, v in rdbg['stageii_errs'].items():
                assert np.allclose(dbg['stageii_errs'][k], v, rtol=1e-7, atol=1e-10), k


def test_other_kernel_shape_is_refused(tmp_path):
    """SMPL-H with one marker less next to SMPL-H: Mosh2Error naming the field."""
    subs = _subjects(str(tmp_path), [(10,), (12,)])
    a, b = subs[0]['case'], subs[1]['case']
    pa, opts, _ = chmosh.prepare_stageii(a['cfg'], **_stagei_outputs(a))
    pb, _, _ = chmosh.prepare_stageii(b['cfg'], b['markers_latent'][:-1], b['latent_labels'][:-1], b['betas'], b['marker_meta'])
    ma, mb = lib.Model(pa, device=0), lib.Model(pb, device=0)
    try:
        with pytest.raises(lib.Mosh2Error, match='n_markers differs'):
            lib.multi_job([ma, mb], [0, 1], [10, 12], opts)
    finally:
        ma.close()
        mb.close()


def _compare_pickles(got, want, exact):
    for k in ('fullpose', 'trans', 'betas'):
        if exact:
            assert np.array_equal(got[k], want[k]), k
    gd, wd = got['stageii_debug_details'], want['stageii_debug_details']
    assert set(got) == set(want) and set(gd) == set(wd) and set(gd['stageii_errs']) == set(wd['stageii_errs'])
    if exact:
        for k in wd['stageii_errs']:
            assert np.array_equal(gd['stageii_errs'][k], wd['stageii_errs'][k]), k
        assert all(np.array_equal(x, y) for x, y in zip(gd['markers_sim'], wd['markers_sim']))
    else:
        # the fast mode's gates (BASELINE.md section 4): >= 99 % of the frames within 1e-3 rad / 0.1 mm
        body = np.abs(got['fullpose'][:, :66] - want['fullpose'][:, :66]).max(1)
        dtr = np.abs(got['trans'] - want['trans']).max(1)
        assert (body > 1e-3).mean() <= 0.01 and (dtr > 1e-4).mean() <= 0.01 and body.max() < 0.05 and dtr.max() < 2e-3
    assert gd['labels_obs'] == wd['labels_obs'] and gd['mocap_fname'] == wd['mocap_fname']
    cg, cw = copy.deepcopy(gd['cfg']), copy.deepcopy(wd['cfg'])
    for c in (cg, cw):
        c['dirs'] = {k: v for k, v in c['dirs'].items() if k in ('session_subject_subfolders', 'stagei_basename')}
    assert cg == cw


def test_run_moshpp_jobs_writes_what_run_once_writes(tmp_path):
    """run_moshpp_jobs on three subjects x two captures (one subject on a second model file) and one capture with its own
    Stage I (perseq_mosh_stagei): the Stage-II pickles equal those of run_moshpp_once of every job bit for bit when both run
    float64 sequentially, lie within the fast-mode gates of run_moshpp_once's in the default mode (whose chunks are planned
    per capture), and a second run launches nothing."""
    from moshpp_b200 import mosh_head, stagei
    subs = _subjects(str(tmp_path / 'synth'), [(60, 45), (50, 40), (40, 55), (48,)])
    root = tmp_path / 'mocap' / 'DS'
    jobs = []
    for k, s in enumerate(subs):
        sess = root / f'subj{k}'
        sess.mkdir(parents=True)
        (sess / 'settings.json').write_text(json.dumps({'gender': 'male'}))
        c = s['case']['cfg']
        base = {'dirs.support_base_dir': str(tmp_path / 'support'), 'surface_model.type': 'smplh',
                'surface_model.fname': c.surface_model.fname, 'moshpp.pose_body_prior_fname': c.moshpp.pose_body_prior_fname,
                'moshpp.pose_hand_prior_fname': c.moshpp.pose_hand_prior_fname, 'moshpp.optimize_fingers': True,
                'moshpp.head_marker_corr_fname': None, 'moshpp.stagei_frame_picker.num_frames': 4,
                'moshpp.stagei_frame_picker.least_avail_markers': 0.8, 'opt_settings.maxiter': 4}
        if k == 3:
            base['moshpp.perseq_mosh_stagei'] = True
        for j, fn in enumerate(s['fnames']):
            dst = str(sess / f'take_{j}.npz')
            shutil.copy(fn, dst)
            jobs.append(dict(base, **{'mocap.fname': dst}))
    meta = subs[0]['case']['marker_meta']

    def at(w):
        out = []
        for job in jobs:
            d = dict(job, **{'dirs.work_base_dir': str(tmp_path / w)})
            cfg = mosh_head.prepare_cfg(**d)
            if not os.path.exists(cfg.dirs.marker_layout.fname):
                os.makedirs(os.path.dirname(cfg.dirs.marker_layout.fname), exist_ok=True)
                stagei.write_marker_layout(cfg.dirs.marker_layout.fname, meta)
            out.append(d)
        return out

    exact_once = functools.partial(chmosh.mosh_stageii, precision='f64', chunk_len=0)
    np.random.seed(0)
    heads = mosh_head.run_moshpp_jobs(at('w_jobs'), stageii_subjects_func=functools.partial(chmosh.mosh_stageii_subjects,
                                                                                             precision='f64', chunk_len=0))
    assert len({h.stagei_fname for h in heads}) == 4 and all(os.path.exists(h.stageii_fname) for h in heads)
    for w in ('w_once', 'w_fast', 'w_once_fast'):         # one Stage I for every run
        for h in heads:
            dst = h.stagei_fname.replace('w_jobs', w)
            os.makedirs(os.path.dirname(dst), exist_ok=True)
            shutil.copy(h.stagei_fname, dst)
    fast = mosh_head.run_moshpp_jobs(at('w_fast'))
    launches = {f.stageii_data['stageii_debug_details']['b200']['batch']['launches'] for f in fast}
    assert launches == {1}
    for h, f, job, job_fast in zip(heads, fast, at('w_once'), at('w_once_fast')):
        one = mosh_head.run_moshpp_once(job, stageii_func=exact_once)
        with open(h.stageii_fname, 'rb') as fh:
            _compare_pickles(pickle.load(fh), one.stageii_data, exact=True)
        one_fast = mosh_head.run_moshpp_once(job_fast)
        with open(f.stageii_fname, 'rb') as fh:
            _compare_pickles(pickle.load(fh), one_fast.stageii_data, exact=False)

    def spy(*a, **kw):
        raise AssertionError('a cached stage was run again')
    again = mosh_head.run_moshpp_jobs(at('w_jobs'), stagei_func=spy, stageii_subjects_func=spy)
    assert all(h.stageii_data is not None for h in again)
