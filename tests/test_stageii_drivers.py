"""The three Stage-II entry points on the CPU: chmosh.mosh_stageii (one capture), mosh_stageii_batch (one subject's captures in
one launch) and mosh_stageii_subjects (several subjects in one multi-model launch), with the library's Model / multi_job
replaced by a job on the single-thread host build of the device source (tests/emu).  Every capture's dictionary from the two
batched entry points equals the one from mosh_stageii, bit for bit; one capture equals the float64 oracle; and the keys of
``stageii_debug_details['b200']`` are those written out here.  The GPU twins are test_gpu_subject_batch.py and
test_gpu_multi_subject.py."""
import ctypes as C

import numpy as np
import pytest

from moshpp_b200 import build, chmosh, lib, synth

SINGLE_KEYS = {'kernel_ms', 'wall_s', 'chunks', 'chunk_len', 'chunk_warmup', 'warmup_full', 'first_extra', 'precision', 'mode',
               'boundary_check', 'totals', 'host_ms', 'subject_cache_hit', 'device_adapter', 'h2d_bytes', 'status', 'counters',
               'pose_reduced', 'frame_ids'}
HOST_MS_KEYS = {'read_mocap_ms', 'prepare_ms', 'dense_view_ms', 'model_create_ms', 'job_create_ms', 'solve_ms', 'overlapped_host_ms',
                'close_ms', 'assemble_ms'}
BATCH_KEYS = {'batch', 'batch_index', 'frame_offset', 'device_adapter', 'status', 'counters', 'pose_reduced', 'frame_ids'}
BATCH_LAUNCH_KEYS = {'shared', 'captures', 'frames', 'kernel_ms', 'wall_s', 'chunks', 'chunk_len', 'chunk_warmup', 'warmup_full',
                     'first_extra', 'precision', 'mode', 'boundary_check', 'totals', 'subject_cache_hit'}
SUBJECTS_KEYS = BATCH_KEYS | {'subject_index'}
SUBJECTS_LAUNCH_KEYS = {'shared', 'launch', 'launches', 'subjects', 'captures', 'frames', 'kernel_ms', 'wall_s', 'chunks', 'chunk_len',
                        'chunk_warmup', 'warmup_full', 'first_extra', 'precision', 'mode', 'boundary_check', 'totals',
                        'subject_cache_hits'}


class _Emu:
    handle = None

    @classmethod
    def get(cls):
        if cls.handle is None:
            cls.handle = C.CDLL(build.build_emu())
            cls.handle.mosh2_emu_upload_markers_range.argtypes = [
                C.c_int32, C.c_int32, C.c_int32, lib._f64p, lib._u8p, C.c_int32, C.c_int32, lib._f64p, C.c_int32, C.c_int32,
                lib._i32p, C.c_int32, C.c_int32, C.c_double, lib._f64p]
        return cls.handle


class FakeModel:
    """lib.Model without a GPU: holds the pack."""

    def __init__(self, pk, device=0, library_path=None):
        self.pk = pk

    def job(self, n_frames, options, *, chunk_len=0, chunk_warmup=0, warmup_full=-1, precision=lib.MOSH2_F32, first_extra=0):
        counts = np.atleast_1d(n_frames)
        return FakeJob([self], np.zeros(len(counts), dtype=np.int32), counts, options,
                       lib.make_schedule(chunk_len, chunk_warmup, warmup_full, first_extra), precision)

    def close(self):
        pass


def fake_multi_job(models, model_of_seq, counts, options, *, chunk_len=0, chunk_warmup=0, warmup_full=-1, first_extra=0,
                   precision=lib.MOSH2_F32):
    return FakeJob(list(models), model_of_seq, counts, options, lib.make_schedule(chunk_len, chunk_warmup, warmup_full, first_extra),
                   precision)


class FakeJob:
    """lib.Job on the host build: the uploads fill host observations, the launch is mosh2_emu_solve_multi (which equals the batch
    solve bit for bit), and the boundary check finds nothing to repair."""

    def __init__(self, models, model_of_seq, counts, options, schedule, precision):
        self.models, self.options, self.schedule, self.precision = models, options, schedule, precision
        self.counts = np.ascontiguousarray(counts, dtype=np.int32)
        self.model_of_seq = np.ascontiguousarray(model_of_seq, dtype=np.int32)
        self.seq_offsets = np.concatenate([[0], np.cumsum(self.counts)]).astype(np.int64)
        self.n_frames = int(self.counts.sum())
        M = models[0].pk.n_markers
        self.obs = np.zeros((self.n_frames, M, 3))
        self.vis = np.zeros((self.n_frames, M), dtype=np.uint8)
        self.result = lib.ResultArrays(self.n_frames, lib.pack_dims(models[0].pk))

    def upload(self, obs, vis):
        self.obs[:], self.vis[:] = obs, vis

    def upload_markers(self, raw, col_of_marker, frame_start, frame_step, unit_per_metre, rot3x3=None):
        self.upload_markers_range(0, self.n_frames, raw, col_of_marker, frame_start, frame_step, unit_per_metre, rot3x3)

    def upload_markers_range(self, frame0, n, raw, col_of_marker, frame_start, frame_step, unit_per_metre, rot3x3=None):
        raw = np.ascontiguousarray(raw, dtype=np.float64)
        cols = np.ascontiguousarray(col_of_marker, dtype=np.int32)
        rot = None if rot3x3 is None else np.ascontiguousarray(rot3x3, dtype=np.float64).reshape(3, 3)
        rc = _Emu.get().mosh2_emu_upload_markers_range(
            self.precision, self.obs.shape[1], self.n_frames, lib._ptr(self.obs, lib._f64p), lib._ptr(self.vis, lib._u8p), int(frame0),
            int(n), lib._ptr(raw, lib._f64p), raw.shape[0], raw.shape[1], lib._ptr(cols, lib._i32p), int(frame_start), int(frame_step),
            float(unit_per_metre), lib._ptr(rot, lib._f64p) if rot is not None else None)
        assert rc == 0

    def launch(self):
        holders = [lib.DescHolder(m.pk) for m in self.models]
        descs = (C.POINTER(lib.ModelDesc) * len(holders))(*[C.pointer(h.desc) for h in holders])
        rc = _Emu.get().mosh2_emu_solve_multi(descs, len(holders), C.byref(self.options), len(self.counts), lib._ptr(self.counts, lib._i32p),
                                              lib._ptr(self.model_of_seq, lib._i32p), lib._ptr(self.obs, lib._f64p),
                                              lib._ptr(self.vis, lib._u8p), C.byref(self.schedule), self.precision, C.byref(self.result.c))
        assert rc == 0

    def sync(self):
        pass

    def boundary_deltas(self):
        return np.zeros((self.num_chunks, 4))

    def kernel_ms(self):
        return 0.0

    def totals(self):
        return {k: 0 for k in ('iterations', 'evaluations', 'builds', 'minimisations', 'emitted_iterations', 'emitted_evaluations',
                               'emitted_builds', 'emitted_minimisations')}

    @property
    def num_chunks(self):
        s = self.schedule
        return sum(chmosh.count_chunks(int(F), s.chunk_len, s.first_extra) for F in self.counts)

    def chunk_ranges(self):
        s, out = self.schedule, []
        for F, a in zip(self.counts, self.seq_offsets):
            first = s.chunk_len + s.first_extra
            if chmosh.count_chunks(int(F), s.chunk_len, s.first_extra) == 1:
                out.append((a, a + F))
                continue
            out.append((a, a + first))
            out += [(b, min(b + s.chunk_len, a + F)) for b in range(a + first, a + F, s.chunk_len)]
        return np.array(out, dtype=np.int32)

    def download(self):
        return self.result

    def close(self):
        pass


@pytest.fixture
def fake_gpu(monkeypatch):
    monkeypatch.setattr(lib, 'Model', FakeModel)
    monkeypatch.setattr(lib, 'multi_job', fake_multi_job)
    chmosh.clear_subject_cache()
    yield
    chmosh.clear_subject_cache()


def _with_duplicate_label(src, dst):
    """A copy of a capture whose first label owns two columns: it takes the host adapter."""
    z = np.load(src)
    mk, labels = z['markers'], list(z['labels'])
    extra = mk[:, :1].copy()
    extra[::3] = np.nan
    np.savez(dst, markers=np.concatenate([mk, extra], 1), labels=np.array(labels + [labels[0]]), frame_rate=120.0)
    return dst


@pytest.fixture(scope='module')
def subjects(tmp_path_factory):
    """Two small SMPL-H subjects, the second on another model file; the first's second capture takes the host adapter."""
    root = tmp_path_factory.mktemp('drivers')
    out = []
    for k, frames in enumerate([(9, 7), (8, 6)]):
        case, fnames = synth.make_subject(str(root), 'C2', frames, n_verts=1500, seq_idx=k, model_seed=k)
        out.append(dict(case=case, fnames=fnames))
    out[0]['fnames'][1] = _with_duplicate_label(out[0]['fnames'][1], str(root / 'dup.npz'))
    return out


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
    assert np.array_equal(ba['pose_reduced'], bb['pose_reduced']) and ba['device_adapter'] == bb['device_adapter']


@pytest.mark.parametrize('schedule', ['sequential_f64', 'chunked_f32'])
def test_entry_points_agree(subjects, fake_gpu, schedule):
    kw = dict(precision='f64', chunk_len=0) if schedule == 'sequential_f64' else \
        dict(precision='f32', chunk_len=4, chunk_warmup=3, warmup_full=2)
    single = [[chmosh.mosh_stageii(fn, *_args(s['case']), **kw) for fn in s['fnames']] for s in subjects]
    batch = [chmosh.mosh_stageii_batch(s['fnames'], *_args(s['case']), **kw) for s in subjects]
    multi = chmosh.mosh_stageii_subjects([dict(cfg=s['case']['cfg'], mocap_fnames=s['fnames'], markers_latent=s['case']['markers_latent'],
                                               latent_labels=s['case']['latent_labels'], betas=s['case']['betas'],
                                               marker_meta=s['case']['marker_meta']) for s in subjects], **kw)
    assert [[o['stageii_debug_details']['b200']['device_adapter'] for o in so] for so in single] == [[True, False], [True, True]]
    for k in range(len(subjects)):
        for one, b, m in zip(single[k], batch[k], multi[k]):
            _assert_same(b, one)
            _assert_same(m, one)

    for so in single:
        for o in so:
            b = o['stageii_debug_details']['b200']
            assert set(b) == SINGLE_KEYS and set(b['host_ms']) == HOST_MS_KEYS
            assert b['precision'] == kw['precision'] and b['chunk_len'] == kw['chunk_len']
    for k, bo in enumerate(batch):
        for q, o in enumerate(bo):
            b = o['stageii_debug_details']['b200']
            assert set(b) == BATCH_KEYS and set(b['batch']) == BATCH_LAUNCH_KEYS
            assert b['batch_index'] == q and b['batch'] is bo[0]['stageii_debug_details']['b200']['batch']
            assert b['batch']['captures'] == 2 and b['batch']['frames'] == sum(len(x['fullpose']) for x in single[k])
    launch = multi[0][0]['stageii_debug_details']['b200']['batch']
    assert launch['launches'] == 1 and launch['subjects'] == 2 and launch['captures'] == 4
    for k, mo in enumerate(multi):
        for c, o in enumerate(mo):
            b = o['stageii_debug_details']['b200']
            assert set(b) == SUBJECTS_KEYS and set(b['batch']) == SUBJECTS_LAUNCH_KEYS and b['batch'] is launch
            assert b['subject_index'] == k and b['batch_index'] == 2 * k + c

    if schedule == 'sequential_f64':
        from oracle import stageii as oracle_stageii
        s = subjects[1]
        c, o = s['case'], single[1][0]
        ref = oracle_stageii.mosh_stageii(s['fnames'][0], *_args(c))
        dbg, rdbg = o['stageii_debug_details'], ref['stageii_debug_details']
        assert np.array_equal(dbg['b200']['frame_ids'], rdbg['frame_ids'])
        assert np.abs(dbg['b200']['pose_reduced'] - ref['_pose_reduced']).max() < 1e-8
        assert np.abs(o['fullpose'] - ref['fullpose']).max() < 1e-8
        assert np.abs(o['trans'] - ref['trans']).max() < 1e-9
        for k, v in rdbg['stageii_errs'].items():
            assert np.allclose(dbg['stageii_errs'][k], v, rtol=1e-7, atol=1e-10), k
