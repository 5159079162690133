"""Several subjects in one launch, on the CPU: the multi-model job (mosh2_job_create_multi) through the single-thread host build
of the device source against each subject solved alone, the grouping of subjects into launches (chmosh.mosh_stageii_subjects),
and the reference's jobs filter (mosh_head.universal_mosh_jobs_filter) on a constructed job tree."""
import ctypes as C
import json
import os
import pickle

import numpy as np
import pytest

from moshpp_b200 import build, chmosh, lib, mosh_head, synth
from moshpp_b200.mocap_interface import MocapSession

# three SMPL-H subjects: other shapes and latent markers (seq_idx), the third on a second model file; captures of few frames
SUBJECTS = [dict(seq_idx=0, model_seed=0, frames=(9, 7)), dict(seq_idx=1, model_seed=0, frames=(8,)),
            dict(seq_idx=2, model_seed=1, frames=(6, 10))]


@pytest.fixture(scope='module')
def subjects(tmp_path_factory):
    root = str(tmp_path_factory.mktemp('multi'))
    out = []
    for s in SUBJECTS:
        case, fnames = synth.make_subject(root, 'C2', s['frames'], n_verts=1500, seq_idx=s['seq_idx'], model_seed=s['model_seed'])
        obs_vis = []
        for fn in fnames:
            m = MocapSession(fn, case['cfg'].mocap.unit)
            obs_vis.append(m.frames_for_labels(case['latent_labels'], range(len(m))))
        out.append(dict(case=case, fnames=fnames, obs_vis=obs_vis))
    return out


@pytest.fixture(scope='module')
def emu_lib():
    return C.CDLL(build.build_emu())


def _options(case):
    pk, cfg = case['pack'], case['cfg']
    return lib.make_options(cfg.opt_settings.weights, optimize_fingers=cfg.moshpp.optimize_fingers and pk.finger_hi > pk.finger_lo)


def _arrays(obs_vis):
    obs = np.ascontiguousarray(np.concatenate([o for o, _ in obs_vis]), dtype=np.float64)
    vis = np.ascontiguousarray(np.concatenate([v for _, v in obs_vis]), dtype=np.uint8)
    return obs, vis


def _solve_batch(handle, case, obs_vis, sched, precision):
    h = lib.DescHolder(case['pack'])
    counts = np.array([len(o) for o, _ in obs_vis], dtype=np.int32)
    obs, vis = _arrays(obs_vis)
    res = lib.ResultArrays(int(counts.sum()), lib.pack_dims(case['pack']))
    opt = _options(case)
    assert handle.mosh2_emu_solve_batch(C.byref(h.desc), C.byref(opt), len(counts), lib._ptr(counts, lib._i32p), lib._ptr(obs, lib._f64p),
                                        lib._ptr(vis, lib._u8p), C.byref(sched), precision, C.byref(res.c)) == 0
    return res


def _solve_multi(handle, packs, seqs, sched, precision, opt):
    """seqs: (model index, (obs, vis)) per sequence, in the order of the job's frame axis"""
    holders = [lib.DescHolder(pk) for pk in packs]
    descs = (C.POINTER(lib.ModelDesc) * len(holders))(*[C.pointer(h.desc) for h in holders])
    counts = np.array([len(ov[0]) for _, ov in seqs], dtype=np.int32)
    mos = np.array([k for k, _ in seqs], dtype=np.int32)
    obs, vis = _arrays([ov for _, ov in seqs])
    res = lib.ResultArrays(int(counts.sum()), lib.pack_dims(packs[0]))
    rc = handle.mosh2_emu_solve_multi(descs, len(holders), C.byref(opt), len(counts), lib._ptr(counts, lib._i32p), lib._ptr(mos, lib._i32p),
                                      lib._ptr(obs, lib._f64p), lib._ptr(vis, lib._u8p), C.byref(sched), precision, C.byref(res.c))
    return rc, res, counts


@pytest.mark.parametrize('precision', [lib.MOSH2_F64, lib.MOSH2_F32])
def test_multi_job_equals_each_subject_alone(subjects, emu_lib, precision):
    """A chunked multi-model job whose sequences of three subjects are interleaved on the frame axis: every sequence's rows
    equal those of its subject's own batch job, bit for bit."""
    packs = [s['case']['pack'] for s in subjects]
    assert len({chmosh.kernel_shape_key(pk) for pk in packs}) == 1
    assert not np.array_equal(packs[0].v0, packs[1].v0) and not np.array_equal(packs[0].coefs, packs[1].coefs)
    assert not np.array_equal(packs[0].j0, packs[2].j0)             # (another model file)
    order = [(0, 0), (1, 0), (2, 0), (0, 1), (2, 1)]                 # (subject, capture)
    sched = lib.make_schedule(chunk_len=4, chunk_warmup=3, warmup_full=2, first_extra=2)
    rc, multi, counts = _solve_multi(emu_lib, packs, [(k, subjects[k]['obs_vis'][c]) for k, c in order], sched, precision,
                                     _options(subjects[0]['case']))
    assert rc == 0
    alone = [_solve_batch(emu_lib, s['case'], s['obs_vis'], sched, precision) for s in subjects]
    offs = np.concatenate([[0], np.cumsum(counts)])
    for q, (k, c) in enumerate(order):
        own = np.concatenate([[0], np.cumsum([len(o) for o, _ in subjects[k]['obs_vis']])])
        a, b = slice(offs[q], offs[q + 1]), slice(own[c], own[c + 1])
        assert (multi.status[a] & lib.ST_SOLVED).any()
        for name in ('fullpose', 'pose', 'trans', 'markers_sim', 'errs', 'status', 'counters'):
            assert np.array_equal(getattr(multi, name)[a], getattr(alone[k], name)[b]), (q, name)


def test_multi_job_refuses_other_kernel_shape(subjects, emu_lib):
    """A pack with one marker less has another kernel shape: the host build refuses the job, and the launch grouping keeps it
    apart."""
    case = subjects[0]['case']
    pk, _, _ = chmosh.prepare_stageii(case['cfg'], case['markers_latent'][:-1], case['latent_labels'][:-1], case['betas'],
                                      case['marker_meta'])
    assert chmosh.kernel_shape_key(pk) != chmosh.kernel_shape_key(case['pack'])
    rc, _, _ = _solve_multi(emu_lib, [case['pack'], pk], [(0, subjects[0]['obs_vis'][0]), (1, subjects[1]['obs_vis'][0])],
                            lib.make_schedule(), lib.MOSH2_F64, _options(case))     # (refused before the observations are read)
    assert rc == -1


def test_launch_grouping(subjects, tmp_path):
    """Subjects share a launch when their kernel shape, options and default schedule are equal: the three SMPL-H subjects
    (two model files) do; a subject with other Stage-II weights, one with another marker count, and a DMPL subject (float64
    exact preset) each get a launch of their own."""
    keys = []
    for s in subjects:
        pk, opts, _ = chmosh.prepare_stageii(s['case']['cfg'], *[s['case'][k] for k in ('markers_latent', 'latent_labels', 'betas', 'marker_meta')])
        keys.append(chmosh.subject_launch_key(pk, opts))
    case = subjects[0]['case']
    heavy = lib.make_options(dict(case['cfg'].opt_settings.weights, stageii_wt_velo=5.0))
    keys.append(chmosh.subject_launch_key(case['pack'], heavy))
    pk, opts, _ = chmosh.prepare_stageii(case['cfg'], case['markers_latent'][:-1], case['latent_labels'][:-1], case['betas'],
                                         case['marker_meta'])
    keys.append(chmosh.subject_launch_key(pk, opts))
    dm = synth.make_case(str(tmp_path), 'C3', frames=6, n_verts=2000)
    pk, opts, _ = chmosh.prepare_stageii(dm['cfg'], dm['markers_latent'], dm['latent_labels'], dm['betas'], dm['marker_meta'])
    assert chmosh.default_schedule(pk.model_type, 'fast', pk.n_dmpl)[2] == 'f64'
    keys.append(chmosh.subject_launch_key(pk, opts))
    keys.append(keys[1])
    assert chmosh.launch_groups(keys) == [[0, 1, 2, 6], [3], [4], [5]]


def _capture(path, labels):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    np.savez(path, markers=np.ones((3, len(labels), 3)), labels=np.array(labels), frame_rate=100.0)
    return path


def _touch(fname):
    os.makedirs(os.path.dirname(fname), exist_ok=True)
    with open(fname, 'wb') as f:
        pickle.dump({}, f)


def test_jobs_filter(tmp_path):
    """universal_mosh_jobs_filter on a job tree of four sessions: finished captures are dropped; of a subject without Stage I
    only the first capture stays (unless every capture determines its own shape); per-capture Stage I (perseq_mosh_stagei) and
    the subjects of a multi-subject capture are keys of their own; only_stagei drops the jobs whose Stage I exists."""
    root = str(tmp_path)
    work = os.path.join(root, 'work')

    def job(fn, **kw):
        return dict({'mocap.fname': fn, 'dirs.work_base_dir': work, 'dirs.support_base_dir': os.path.join(root, 'support')}, **kw)

    done = [_capture(f'{root}/mocap/DS/done/take{k}.npz', ['A', 'B']) for k in range(3)]      # Stage I and take0's Stage II exist
    fresh = [_capture(f'{root}/mocap/DS/fresh/take{k}.npz', ['A', 'B']) for k in range(3)]    # nothing exists yet
    perseq = [_capture(f'{root}/mocap/DS/perseq/take{k}.npz', ['A', 'B']) for k in range(2)]
    duo = _capture(f'{root}/mocap/DS/duo/dance.npz', ['bob:A', 'bob:B', 'alice:A', 'alice:B'])
    for d in ('done', 'fresh', 'perseq'):
        with open(f'{root}/mocap/DS/{d}/settings.json', 'w') as f:
            json.dump({'gender': 'male'}, f)
    with open(f'{root}/mocap/DS/duo/settings.json', 'w') as f:
        json.dump({'alice': {'gender': 'female'}, 'bob': {'gender': 'male'}}, f)
    _touch(f'{work}/DS/done/male_stagei.pkl')
    _touch(f'{work}/DS/done/take0_stageii.pkl')
    _touch(f'{work}/DS/duo/bob/male_stagei.pkl')
    jobs = ([job(fn) for fn in done] + [job(fn) for fn in fresh] + [job(fn, **{'moshpp.perseq_mosh_stagei': True}) for fn in perseq]
            + [job(duo, **{'mocap.subject_id': i}) for i in (0, 1)])
    names = lambda js: [(os.path.basename(j['mocap.fname']), j.get('mocap.subject_id')) for j in js]
    assert names(mosh_head.universal_mosh_jobs_filter(jobs)) == [
        ('take1.npz', None), ('take2.npz', None), ('take0.npz', None), ('take0.npz', None), ('take1.npz', None),
        ('dance.npz', 0), ('dance.npz', 1)]
    assert names(mosh_head.universal_mosh_jobs_filter(jobs, determine_shape_for_each_seq=True)) == [
        ('take1.npz', None), ('take2.npz', None), ('take0.npz', None), ('take1.npz', None), ('take2.npz', None),
        ('take0.npz', None), ('take1.npz', None), ('dance.npz', 0), ('dance.npz', 1)]
    assert names(mosh_head.universal_mosh_jobs_filter(jobs, only_stagei=True)) == [
        ('take0.npz', None), ('take0.npz', None), ('take1.npz', None), ('dance.npz', 0)]


def test_run_moshpp_jobs_writes_what_run_once_writes(tmp_path):
    """The dataset head on the CPU (Stage I on the host build of the device source, the float64 oracle as Stage II): two
    subjects x two captures and one capture with its own Stage I.  One Stage-II call for all of them; the pickles equal those
    of run_moshpp_once of every job; a second run loads everything."""
    import functools
    import shutil
    from conftest import EmuStageIBackend
    from moshpp_b200 import stagei
    from oracle import stageii as oracle_stageii

    def oracle(mocap_fname, cfg, markers_latent, latent_labels, betas, marker_meta, v_template_fname=None):
        out = oracle_stageii.mosh_stageii(mocap_fname, cfg, markers_latent, latent_labels, betas, marker_meta, v_template_fname)
        out.pop('_pose_reduced')
        out['stageii_debug_details'].pop('oracle_stats')
        return out

    calls = []

    def subjects_func(subjects):
        calls.append([list(s['mocap_fnames']) for s in subjects])
        return [[oracle(fn, s['cfg'], s['markers_latent'], s['latent_labels'], s['betas'], s['marker_meta'], s.get('v_template_fname'))
                 for fn in s['mocap_fnames']] for s in subjects]

    root = tmp_path / 'mocap' / 'DS'
    jobs = []
    for k, frames in enumerate([(9, 8), (10, 7), (8,)]):
        case, fnames = synth.make_subject(str(tmp_path / 'synth'), 'C2', frames, n_verts=1500, seq_idx=k, model_seed=1 if k == 1 else 0)
        sess = root / f'subj{k}'
        sess.mkdir(parents=True)
        (sess / 'settings.json').write_text(json.dumps({'gender': 'female'}))
        c = case['cfg']
        base = {'dirs.support_base_dir': str(tmp_path / 'support'), 'surface_model.type': 'smplh', 'surface_model.fname': c.surface_model.fname,
                'moshpp.pose_body_prior_fname': c.moshpp.pose_body_prior_fname, 'moshpp.pose_hand_prior_fname': c.moshpp.pose_hand_prior_fname,
                'moshpp.optimize_fingers': True, 'moshpp.head_marker_corr_fname': None, 'moshpp.stagei_frame_picker.num_frames': 4,
                'moshpp.stagei_frame_picker.least_avail_markers': 0.8, 'opt_settings.maxiter': 4, 'moshpp.perseq_mosh_stagei': k == 2}
        for j, fn in enumerate(fnames):
            dst = str(sess / f'take_{j}.npz')
            shutil.copy(fn, dst)
            jobs.append(dict(base, **{'mocap.fname': dst}))
        meta = case['marker_meta']

    def at(w):
        out = []
        for job in jobs:
            d = dict(job, **{'dirs.work_base_dir': str(tmp_path / w)})
            layout = mosh_head.prepare_cfg(**d).dirs.marker_layout.fname
            if not os.path.exists(layout):
                os.makedirs(os.path.dirname(layout), exist_ok=True)
                stagei.write_marker_layout(layout, meta)
            out.append(d)
        return out

    stagei_func = functools.partial(stagei.mosh_stagei, backend=EmuStageIBackend())
    np.random.seed(0)
    heads = mosh_head.run_moshpp_jobs(at('w_jobs'), stagei_func=stagei_func, stageii_subjects_func=subjects_func)
    assert calls == [[[j['mocap.fname'] for j in jobs[:2]], [j['mocap.fname'] for j in jobs[2:4]], [jobs[4]['mocap.fname']]]]
    assert len({h.stagei_fname for h in heads}) == 3
    for h in heads:
        dst = h.stagei_fname.replace('w_jobs', 'w_once')
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        shutil.copy(h.stagei_fname, dst)
    for h, job in zip(heads, at('w_once')):
        one = mosh_head.run_moshpp_once(job, stageii_func=oracle)
        with open(h.stageii_fname, 'rb') as f:
            got = pickle.load(f)
        want = one.stageii_data
        assert set(got) == set(want)
        for k in ('fullpose', 'trans', 'betas', 'markers_latent'):
            assert np.array_equal(got[k], want[k]), k
        gd, wd = got['stageii_debug_details'], want['stageii_debug_details']
        assert set(gd) == set(wd) and gd['labels_obs'] == wd['labels_obs'] and gd['mocap_fname'] == wd['mocap_fname']
        for k in wd['stageii_errs']:
            assert np.array_equal(gd['stageii_errs'][k], wd['stageii_errs'][k]), k
        strip = lambda c: dict(c, dirs={k: v for k, v in c['dirs'].items() if k in ('session_subject_subfolders', 'stagei_basename')})
        assert strip(gd['cfg']) == strip(wd['cfg'])

    def spy(*a, **kw):
        raise AssertionError('a cached stage was run again')
    again = mosh_head.run_moshpp_jobs(at('w_jobs'), stagei_func=spy, stageii_subjects_func=spy)
    assert all(h.stageii_data is not None for h in again)
