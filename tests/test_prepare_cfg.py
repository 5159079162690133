"""cfg.prepare_cfg: moshpp_conf.yaml and its omegaconf resolvers (tools/run_tools.py:88-183) restated as plain functions --
paths, names and gender derived from the capture path, for one subject, several subjects with `subject_id`, and
`perseq_mosh_stagei`; explicit values win over derived ones; missing inputs raise."""
import json
import os

import numpy as np
import pytest

from moshpp_b200.cfg import MissingMandatoryValue, prepare_cfg


def _capture(path, labels):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    np.savez(path, markers=np.ones((3, len(labels), 3)), labels=np.array(labels), frame_rate=100.0)
    return path


@pytest.fixture()
def tree(tmp_path):
    root = str(tmp_path)
    single = _capture(os.path.join(root, 'mocap', 'My DS', 'sess 01', 'walk fast.01.npz'), ['LFHD', 'RFHD', 'C7'])
    with open(os.path.join(os.path.dirname(single), 'settings.json'), 'w') as f:
        json.dump({'gender': 'female'}, f)
    multi = _capture(os.path.join(root, 'mocap', 'DS2', 'duo', 'dance.npz'), ['bob:LFHD', 'bob:C7', 'alice:LFHD', 'alice:C7'])
    with open(os.path.join(os.path.dirname(multi), 'settings.json'), 'w') as f:
        json.dump({'alice': {'gender': 'female'}, 'bob': {'gender': 'male'}}, f)
    return dict(root=root, single=single, multi=multi, work=os.path.join(root, 'work'), support=os.path.join(root, 'support'))


def test_single_subject(tree):
    w, s = tree['work'], tree['support']
    cfg = prepare_cfg(**{'mocap.fname': tree['single'], 'dirs.work_base_dir': w, 'dirs.support_base_dir': s})
    mc, d = cfg.mocap, cfg.dirs
    assert (mc.ds_name, mc.session_name, mc.basename) == ('MyDS', 'sess01', 'walkfast.01')
    assert mc.subject_names == ['null'] and mc.subject_name is None and mc.multi_subject is False
    assert cfg.surface_model.gender == 'female'
    assert cfg.surface_model.fname == f'{s}/smplx/female/model.pkl' and cfg.surface_model.dmpl_fname == f'{s}/smplx/female/dmpl.pkl'
    assert cfg.moshpp.pose_body_prior_fname == f'{s}/smplx/pose_body_prior.pkl'
    assert cfg.moshpp.pose_hand_prior_fname == f'{s}/smplx/pose_hand_prior.npz'
    assert cfg.moshpp.head_marker_corr_fname == f'{s}/ssm_head_marker_corr.npz'
    assert d.session_subject_subfolders == 'sess01'
    assert d.marker_layout.basename == 'MyDS_smplx' and d.marker_layout.fname == f'{w}/MyDS/MyDS_smplx.json'
    assert d.stagei_basename == 'female' and d.stagei_fname == f'{w}/MyDS/sess01/female_stagei.pkl'
    assert d.stageii_fname == f'{w}/MyDS/sess01/walkfast.01_stageii.pkl' and d.log_fname == f'{w}/MyDS/sess01/walkfast.01.log'
    assert cfg.moshpp.stagei_frame_picker.stagei_mocap_fnames is None
    assert cfg.moshpp.stagei_frame_picker.type == 'random_strict' and cfg.moshpp.stagei_frame_picker.seed == 100
    assert cfg.opt_settings.weights_type == 'smplx' and cfg.opt_settings.weights['stageii_wt_data'] == 400
    assert cfg.runtime.stagei_only is False and cfg.moshpp.betas_fname is None and cfg.moshpp.v_template_fname is None


def test_multi_subject_with_subject_id(tree):
    w = tree['work']
    cfg = prepare_cfg(**{'mocap.fname': tree['multi'], 'mocap.subject_id': 1, 'dirs.work_base_dir': w, 'dirs.support_base_dir': 's'})
    assert cfg.mocap.subject_names == ['alice', 'bob'] and cfg.mocap.subject_name == 'bob' and cfg.mocap.multi_subject
    assert cfg.surface_model.gender == 'male'
    assert cfg.dirs.session_subject_subfolders == 'duo/bob'
    assert cfg.dirs.stagei_fname == f'{w}/DS2/duo/bob/male_stagei.pkl'
    assert cfg.dirs.stageii_fname == f'{w}/DS2/duo/bob/dance_stageii.pkl'
    # subject_id -1: the subject prefixes are ignored, and the gender must then be given at the top of settings.json
    with pytest.raises(FileNotFoundError, match='gender settings not found'):
        prepare_cfg(**{'mocap.fname': tree['multi'], 'dirs.work_base_dir': w, 'dirs.support_base_dir': 's'})


def test_perseq_mosh_stagei(tree):
    w = tree['work']
    cfg = prepare_cfg({'moshpp': {'perseq_mosh_stagei': True}, 'surface_model': {'type': 'smplh'}},
                      **{'mocap.fname': tree['single'], 'dirs.work_base_dir': w, 'dirs.support_base_dir': 's'})
    d = cfg.dirs
    assert cfg.moshpp.stagei_frame_picker.stagei_mocap_fnames == [tree['single']]
    assert d.marker_layout.basename == 'walkfast.01_smplh' and d.marker_layout.fname == f'{w}/MyDS/sess01/walkfast.01_smplh.json'
    assert d.stagei_basename == 'walkfast.01_female' and d.stagei_fname == f'{w}/MyDS/sess01/walkfast.01_female_stagei.pkl'
    assert cfg.opt_settings.weights_type == 'smplh'


def test_merge_order_and_explicit_values_win(tree):
    base = {'mocap.fname': tree['single'], 'dirs.work_base_dir': 'w', 'dirs.support_base_dir': 's'}
    cfg = prepare_cfg({'surface_model': {'gender': 'neutral', 'fname': '/m/model.npz'}, 'dirs': {'stageii_fname': '/x.pkl'},
                       'mocap': {'unit': 'm'}}, **dict(base, **{'mocap.unit': 'cm', 'moshpp.optimize_fingers': 'true',
                                                                'opt_settings.maxiter': '7'}))
    assert cfg.mocap.unit == 'm'                                            # dict_cfg after the dotlist
    assert cfg.moshpp.optimize_fingers is True and cfg.opt_settings.maxiter == 7
    assert cfg.surface_model.gender == 'neutral' and cfg.surface_model.fname == '/m/model.npz'
    assert cfg.dirs.stageii_fname == '/x.pkl'
    assert cfg.dirs.stagei_fname == 'w/MyDS/sess01/neutral_stagei.pkl'     # derived from the explicit gender
    assert cfg.surface_model.dmpl_fname == 's/smplx/neutral/dmpl.pkl'


def test_missing_inputs_raise(tree):
    os.remove(os.path.join(os.path.dirname(tree['single']), 'settings.json'))
    with pytest.raises(FileNotFoundError, match='settings.json'):
        prepare_cfg(**{'mocap.fname': tree['single'], 'dirs.work_base_dir': 'w', 'dirs.support_base_dir': 's'})
    for missing in ('mocap.fname', 'dirs.work_base_dir', 'dirs.support_base_dir'):
        kw = {'mocap.fname': tree['single'], 'dirs.work_base_dir': 'w', 'dirs.support_base_dir': 's', 'surface_model.gender': 'male'}
        del kw[missing]
        with pytest.raises(MissingMandatoryValue, match=missing):
            prepare_cfg(**kw)
