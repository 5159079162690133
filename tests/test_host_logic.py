"""Host-side logic that needs no GPU: result assembly (chmosh.py:712-741), chunk sizing, bench bookkeeping."""
import importlib.util
import os

import numpy as np

from conftest import dense_obs, run_oracle
from moshpp_b200 import chmosh, lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_result_assembly_matches_reference_layout(cases, emu):
    """The dictionary builder is fed with the device-source result arrays (host build) and compared, key by key,
    with the oracle's restatement of chmosh.py:712-741."""
    case = cases('C3')
    obs, vis = dense_obs(case)
    vis = vis.copy()
    vis[4] = False                                   # a frame without markers is dropped from every list
    res = emu(case, obs_vis=(obs, vis))
    pk, opts, flags = chmosh.prepare_stageii(case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])
    data = chmosh.assemble_stageii_data(res, obs, vis, case['latent_labels'], pk, flags, dyn=True)
    n = int(vis.any(1).sum())
    assert data['fullpose'].shape == (n, 165) and data['trans'].shape == (n, 3) and data['dmpls'].shape == (n, 8)
    dbg = data['stageii_debug_details']
    assert len(dbg['markers_sim']) == len(dbg['markers_obs']) == len(dbg['labels_obs']) == n
    for mk, ob, lb in zip(dbg['markers_sim'], dbg['markers_obs'], dbg['labels_obs']):
        assert mk.shape == ob.shape == (len(lb), 3)
    solved = np.nonzero(vis.any(1))[0]
    for k, f in enumerate(solved):                   # the lists are cut out of the right frames, in label order
        assert np.array_equal(dbg['markers_sim'][k], res.markers_sim[f][vis[f]])
        assert np.array_equal(dbg['markers_obs'][k], obs[f][vis[f]])
        assert dbg['labels_obs'][k] == [l for l, v in zip(case['latent_labels'], vis[f]) if v]
    assert np.array_equal(data['fullpose'], res.fullpose[solved]) and np.array_equal(data['trans'], res.trans[solved])
    e = dbg['stageii_errs']
    assert list(e.keys()) == ['data', 'poseB', 'poseH', 'dmpl', 'extrap_dmpl', 'velo']
    assert len(e['data']) == n and len(e['extrap_dmpl']) == n - 1 and len(e['velo']) == n - 2
    # same numbers as the oracle on the unmodified visibility
    ref = run_oracle(case)
    res2 = emu(case)
    d2 = chmosh.assemble_stageii_data(res2, *dense_obs(case), case['latent_labels'], pk, flags, dyn=True)
    for k, v in ref['stageii_debug_details']['stageii_errs'].items():
        assert np.allclose(d2['stageii_debug_details']['stageii_errs'][k], v, rtol=1e-8, atol=1e-12)
    assert np.abs(d2['fullpose'] - ref['fullpose']).max() < 1e-9


def test_auto_chunk_len():
    assert chmosh.auto_chunk_len(500) == 4 and chmosh.auto_chunk_len(4000) == 31 and chmosh.auto_chunk_len(12) == 4
    assert chmosh.auto_chunk_len(4000, sm_budget=37) == 109


def test_planned_schedule_counts_chunks_like_the_chunk_table():
    """chmosh.count_chunks mirrors mosh2_host::chunk_table (incl. the longer first chunk), and the plan of the north-star
    sequence fills the SMs with one wave."""
    def brute(F, L, E):
        if L <= 0 or L >= F:
            return 1
        n, f = 0, 0
        while f < F:
            f += L + (E if f == 0 else 0)
            n += 1
        return n
    for F in (1, 5, 57, 500, 4000):
        for L in (0, 1, 4, 27, 56, 4000):
            for E in (0, 3, 52):
                assert chmosh.count_chunks(F, L, E) == brute(F, L, E), (F, L, E)
    assert chmosh.first_chunk_extra(64, 48) == 52 and chmosh.first_chunk_extra(256, -1) == 256 and chmosh.first_chunk_extra(0, 0) == 0
    S = chmosh.NUM_SMS
    L = chmosh.plan_chunk_len([4000], S, 64, 48, first_extra=52)
    assert L == 30 and chmosh.count_chunks(4000, L, 52) <= S < chmosh.count_chunks(4000, L - 1, 52)
    L5 = chmosh.plan_chunk_len([4000] * 32, S, 64, 48, first_extra=52)
    assert sum(chmosh.count_chunks(4000, L5, 52) for _ in range(32)) <= 2 * S


def test_options_follow_the_config(cases):
    case = cases('C2')
    pk, opts, flags = chmosh.prepare_stageii(case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])
    assert (opts.wt_data, opts.wt_poseB, opts.wt_velo, opts.wt_annealing, opts.maxiter) == (400.0, 1.6, 2.5, 2.5, 100)
    assert opts.optimize_fingers == 1 and opts.optimize_dynamics == 0
    # fingers are switched off when the layout has no finger markers (chmosh.py:475-486)
    c1 = cases('C1')
    c1['cfg'].moshpp.optimize_fingers = True
    _, o1, f1 = chmosh.prepare_stageii(c1['cfg'], c1['markers_latent'], c1['latent_labels'], c1['betas'], c1['marker_meta'])
    assert not f1['optimize_fingers'] and o1.optimize_fingers == 0 and c1['cfg'].moshpp.optimize_fingers is False


def test_bench_algorithmic_bytes_match_baseline_table(cases):
    """BASELINE.md section 3: C2 R=385 n=111 B_K1=174.1 KB B_K2=197.8 KB."""
    spec = importlib.util.spec_from_file_location('bench', os.path.join(ROOT, 'bench.py'))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    ab = bench.algorithmic_bytes(cases('C2')['pack'])
    assert (ab['R'], ab['n']) == (385, 111)
    assert round(ab['B_K1'] / 1000, 1) == 174.1 and round(ab['B_K2'] / 1000, 1) == 197.8
    ab3 = bench.algorithmic_bytes(cases('C3')['pack'])
    assert (ab3['R'], ab3['n']) == (452, 119)


def test_amass_writer_round_trip(cases, emu, tmp_path):
    """pkl merge + AMASS npz layout (mosh_head.py:289-295,444-541; run_tools.py:70-85)."""
    from moshpp_b200 import amass_io
    case = cases('C3')
    obs, vis = dense_obs(case)
    pk, opts, flags = chmosh.prepare_stageii(case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])
    data = chmosh.assemble_stageii_data(emu(case), obs, vis, case['latent_labels'], pk, flags, dyn=True)
    data['stageii_debug_details'].update(markers_orig=obs, labels_orig=case['latent_labels'], mocap_frame_rate=120.0,
                                         mocap_time_length=len(obs) / 120.0)
    stagei = dict(markers_latent=case['markers_latent'], latent_labels=case['latent_labels'], betas=case['betas'],
                  marker_meta=case['marker_meta'], markers_latent_vids={l: 0 for l in case['latent_labels']})
    merged = amass_io.merge_stageii(data, stagei, case['cfg'], 1.5, str(tmp_path / 'x_stageii.pkl'))
    assert merged['stageii_debug_details']['stageii_elapsed_time'] == 1.5 and 'betas' in merged
    npz = amass_io.load_as_amass_npz(str(tmp_path / 'x_stageii.pkl'), str(tmp_path / 'x_stageii.npz'), include_markers=True)
    n = len(merged['fullpose'])
    assert npz['poses'].shape == (n, 165) and npz['root_orient'].shape == (n, 3) and npz['pose_body'].shape == (n, 63)
    assert npz['pose_jaw'].shape == (n, 3) and npz['pose_eye'].shape == (n, 6) and npz['pose_hand'].shape == (n, 90)
    assert npz['dmpls'].shape == (n, 8) and npz['betas'].shape == (16,) and npz['surface_model_type'] == 'smplx'
    back = np.load(str(tmp_path / 'x_stageii.npz'), allow_pickle=True)
    assert np.array_equal(back['trans'], merged['trans']) and back['num_markers'] == 67
    # the per-subject file next to it (mosh_head.py:521-537): the Stage-I keys only, written once
    s1 = np.load(str(tmp_path / f"{npz['gender']}_stagei.npz"), allow_pickle=True)
    assert set(s1.files) == {'gender', 'surface_model_type', 'markers_latent', 'latent_labels', 'markers_latent_vids', 'betas'}
    assert np.array_equal(s1['markers_latent'], case['markers_latent']) and s1['betas'].shape == (16,)
    merged['stagei_debug_details'] = {'v_template': np.zeros((5, 3))}
    more = amass_io.load_as_amass_npz(merged, str(tmp_path / 'y_stageii.npz'), str(tmp_path / 'sub' / 'subject_stagei.npz'),
                                      include_extra_details=True)
    assert more['surface_model_fname'] == case['cfg'].surface_model.fname and more['v_template'].shape == (5, 3)
    assert 'v_template' in np.load(str(tmp_path / 'sub' / 'subject_stagei.npz'), allow_pickle=True).files
    assert 'markers' not in more
    parts = amass_io.turn_fullpose_into_parts(np.zeros((2, 48)), 'mano')
    assert parts['pose_hand'].shape == (2, 45) and 'pose_body' not in parts


def test_synonym_labels_are_resolved_like_the_reference(cases, tmp_path):
    """The reference builds its Stage-II MocapSession with labels_map=general_labels_map (chmosh.py:466): a capture that
    names markers HEAD_TOP / L_ANK / ... must yield the same dense observations as one with the canonical names."""
    from moshpp_b200.mocap_interface import MocapSession, general_labels_map
    table = general_labels_map()
    assert table['HEAD_TOP'] == 'ARIEL' and table['L_ANK'] == 'LANK' and table['MIDBACK'] == 'T8' and len(table) >= 190
    case = cases('C1')
    z = np.load(case['mocap_fname'].replace('.c3d', '.npz')) if case['mocap_fname'].endswith('.npz') else None
    ref = MocapSession(case['mocap_fname'], 'mm')
    obs0, vis0 = ref.frames_for_labels(case['latent_labels'], range(len(ref)))
    # rename every column that has a synonym to (one of) its raw spellings, with a subject prefix and a blank
    inverse = {}
    for raw, canon in table.items():
        inverse.setdefault(canon, raw)
    raw_labels = ['subj:' + inverse.get(l, l).replace('_', '_ ', 1) for l in ref.labels]
    renamed = sum(1 for l in ref.labels if l in inverse)
    assert renamed >= 10
    fn = str(tmp_path / 'synonyms.npz')
    np.savez(fn, markers=ref.markers * 1000.0, labels=np.array(raw_labels), frame_rate=120.0)
    obs1, vis1 = MocapSession(fn, 'mm').frames_for_labels(case['latent_labels'], range(len(ref)))
    assert np.array_equal(vis0, vis1) and np.allclose(obs0, obs1, atol=1e-12)
    # opt-out: raw labels -> the renamed markers are invisible
    _, vis2 = MocapSession(fn, 'mm', labels_map=None).frames_for_labels(case['latent_labels'], range(len(ref)))
    assert vis2.sum() < vis1.sum()


def test_duplicate_labels_take_the_last_available_sample(tmp_path):
    """markers_asdict writes a frame's dictionary in column order and only for available samples
    (tools/mocap_interface.py:262-271): of two columns with one label the last AVAILABLE one wins, per frame."""
    from moshpp_b200.mocap_interface import MocapSession
    from oracle.stageii import frames_from_mocap
    mk = np.zeros((3, 3, 3))
    mk[:, 0] = [[1, 1, 1], [2, 2, 2], [3, 3, 3]]                 # A, always there
    mk[:, 1] = [[10, 10, 10], [np.nan, 0, 0], [0, 0, 0]]         # A again: present, NaN, all-zero
    mk[:, 2] = [[7, 7, 7], [8, 8, 8], [9, 9, 9]]                 # B
    fn = str(tmp_path / 'dup.npz')
    np.savez(fn, markers=mk, labels=np.array(['A', 'A', 'B']), frame_rate=100.0)
    s = MocapSession(fn, 'm')
    obs, vis = s.frames_for_labels(['A', 'B', 'C'], range(3))
    assert vis.tolist() == [[True, True, False]] * 3
    assert obs[:, 0, 0].tolist() == [10.0, 2.0, 3.0] and obs[:, 1, 0].tolist() == [7.0, 8.0, 9.0]
    d = s.markers_asdict()
    assert [float(f['A'][0]) for f in d] == [10.0, 2.0, 3.0]
    fr = frames_from_mocap(s.markers, s.labels, ['A', 'B', 'C'])      # the oracle's restatement of the same rule
    assert [float(f[1][0, 0]) for f in fr] == [10.0, 2.0, 3.0]


def test_model_pickles_with_chumpy_leaves_load_without_chumpy(cases, tmp_path):
    """The released SMPL-family files hold chumpy objects (``chumpy.ch.Ch`` leaves with the array under ``x``) and scipy
    sparse matrices pickled under old module paths; the reference reads them through chumpy
    (smpl_fast_derivatives.py:61,149-166).  The loader resolves them to plain arrays without chumpy being installed and
    the resulting SurfaceModel equals the one read from a plain-array pickle."""
    import pickle
    import sys
    import types
    import scipy.sparse as sp
    from moshpp_b200 import pack
    case = cases('C2')
    sm = case['cfg'].surface_model
    with open(sm.fname, 'rb') as f:
        dd = pickle.load(f)
    assert 'chumpy' not in sys.modules
    mod, sub = types.ModuleType('chumpy'), types.ModuleType('chumpy.ch')

    class Ch:                                       # what pickle records: the class path and the instance dict
        def __init__(self, x):
            self.x = np.asarray(x)
            self._dirty_vars = set()
    Ch.__module__, Ch.__qualname__ = 'chumpy.ch', 'Ch'
    sub.Ch = Ch
    mod.ch = sub
    sys.modules['chumpy'], sys.modules['chumpy.ch'] = mod, sub
    try:
        chd = dict(dd)
        for k in ('v_template', 'shapedirs', 'posedirs', 'weights'):
            chd[k] = Ch(dd[k])
        chd['J_regressor'] = sp.csc_matrix(np.asarray(dd['J_regressor'].toarray() if hasattr(dd['J_regressor'], 'toarray') else dd['J_regressor']))
        fname = str(tmp_path / 'model_ch.pkl')
        with open(fname, 'wb') as f:
            pickle.dump(chd, f, protocol=2)
    finally:
        del sys.modules['chumpy'], sys.modules['chumpy.ch']
    try:
        with open(fname, 'rb') as f:
            pickle.load(f)
        raise AssertionError('plain pickle.load was expected to need chumpy')
    except ModuleNotFoundError:
        pass
    kw = dict(pose_hand_prior_fname=case['cfg'].moshpp.pose_hand_prior_fname, use_hands_mean=bool(sm.use_hands_mean),
              dof_per_hand=int(sm.dof_per_hand), surface_model_type=sm.type)
    a = pack.load_surface_model(sm.fname, **kw)
    b = pack.load_surface_model(fname, **kw)
    for k in ('v_template', 'shapedirs', 'posedirs', 'weights', 'J_regressor', 'parents', 'hand_comps', 'hands_mean'):
        assert np.array_equal(getattr(a, k), getattr(b, k)), k
