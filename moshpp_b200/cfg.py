"""Duck-typed configuration without omegaconf (absent here).  ``default_cfg``: the Stage-II-relevant defaults of the
reference's support_data/conf/moshpp_conf.yaml (lines 13-31, 34-50, 95-125); ``prepare_cfg``: the whole yaml with its
interpolations, for the head (``mosh_head.MoSh``).  ``mosh_stageii`` accepts any mapping with attribute/key access
(DictConfig, AttrDict, ...)."""
from __future__ import annotations

import copy


class AttrDict(dict):
    """Minimal attribute/key mapping standing in for omegaconf's DictConfig (absent here)."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __setattr__(self, k, v):
        self[k] = v

    @staticmethod
    def wrap(d):
        if isinstance(d, dict):
            return AttrDict({k: AttrDict.wrap(v) for k, v in d.items()})
        return d


STAGEII_WEIGHTS = dict(stageii_wt_data=400, stageii_wt_velo=2.5, stageii_wt_dmpl=1.0, stageii_wt_expr=1.0,
                       stageii_wt_poseB=1.6, stageii_wt_poseH=1.0, stageii_wt_poseF=1.0, stageii_wt_annealing=2.5)


# Stage I (support_data/conf/moshpp_conf.yaml:99-117, the `smplh` weight block that every surface model type uses by default)
STAGEI_WEIGHTS = dict(stagei_wt_poseH=3.0, stagei_wt_poseF=3., stagei_wt_expr=34., stagei_wt_pose=3., stagei_wt_poseB=3.,
                      stagei_wt_init_finger_left=400.0, stagei_wt_init_finger_right=400.0, stagei_wt_init_finger=400.0,
                      stagei_wt_betas=10., stagei_wt_init=300, stagei_wt_data=75., stagei_wt_surf=10000.,
                      stagei_wt_annealing=[1., .5, .25, .125])


def default_cfg(**over) -> AttrDict:
    """The Stage-II-relevant defaults of support_data/conf/moshpp_conf.yaml (lines 13-31,34-50,95-125)."""
    cfg = AttrDict.wrap({
        'mocap': {'fname': None, 'unit': 'mm', 'rotate': None, 'start_fidx': 0, 'end_fidx': -1, 'ds_rate': 1,
                  'subject_name': 'null', 'multi_subject': False},
        'surface_model': {'type': 'smplx', 'fname': None, 'dmpl_fname': None, 'num_betas': 16,
                          'betas_expr_start_id': 300, 'num_dmpls': 8, 'dof_per_hand': 24, 'num_expressions': 80,
                          'use_hands_mean': True, 'gender': 'neutral'},
        'moshpp': {'pose_body_prior_fname': None, 'pose_hand_prior_fname': None, 'optimize_fingers': False,
                   'optimize_face': False, 'optimize_toes': False, 'optimize_betas': True,
                   'optimize_dynamics': False, 'verbosity': 1},
        'opt_settings': {'weights_type': 'smplh', 'weights': dict(STAGEII_WEIGHTS, **STAGEI_WEIGHTS), 'maxiter': 100,
                         'stagei_lr': 1e-3, 'extra_initial_rigid_adjustment': False},
    })
    for k, v in over.items():
        node = cfg
        parts = k.split('.')
        for q in parts[:-1]:
            node = node[q]
        node[parts[-1]] = v
    return cfg


# ---------------------------------------------------------------------------------------------------------------------
# The whole of support_data/conf/moshpp_conf.yaml, for the head (mosh_head.MoSh).  The yaml's interpolations (omegaconf
# resolvers, tools/run_tools.py:88-183) are restated as plain functions in ``prepare_cfg``; DERIVED marks their places.
# ---------------------------------------------------------------------------------------------------------------------
DERIVED = '<derived>'
MISSING = '???'

_OPT_WEIGHTS_SMPLX = dict(STAGEI_WEIGHTS, **STAGEII_WEIGHTS)

MOSHPP_CONF = {
    'mocap': {'fname': MISSING, 'ds_name': DERIVED, 'subject_id': -1, 'subject_names': DERIVED, 'subject_name': DERIVED,
              'multi_subject': DERIVED, 'session_name': DERIVED, 'basename': DERIVED, 'unit': 'mm', 'rotate': None,
              'exclude_markers': None, 'exclude_marker_types': None, 'only_markers': None, 'start_fidx': 0, 'end_fidx': -1,
              'ds_rate': 1},
    'surface_model': {'type': 'smplx', 'fname': DERIVED, 'dmpl_fname': DERIVED, 'num_betas': 16, 'betas_expr_start_id': 300,
                      'num_dmpls': 8, 'dof_per_hand': 24, 'num_expressions': 80, 'use_hands_mean': True, 'gender': DERIVED},
    'moshpp': {'head_marker_corr_fname': DERIVED, 'pose_body_prior_fname': DERIVED, 'pose_hand_prior_fname': DERIVED,
               'wrist_markers_on_stick': False, 'perseq_mosh_stagei': False, 'optimize_fingers': False, 'optimize_face': False,
               'optimize_toes': False, 'optimize_betas': True, 'optimize_dynamics': False, 'v_template_fname': None,
               'betas_fname': None, 'separate_types': ['body', 'face', 'finger'],
               'stagei_frame_picker': {'type': 'random_strict', 'seed': 100, 'num_frames': 12, 'least_avail_markers': 1.0,
                                       'stagei_mocap_fnames': DERIVED},
               'verbosity': 1,
               'visualization': {'marker_radius': {'body': 0.009, 'face': 0.004, 'finger': 0.005, 'finger_left': 0.005,
                                                   'finger_right': 0.005}}},
    'dirs': {'support_base_dir': MISSING, 'work_base_dir': MISSING, 'session_subject_subfolders': DERIVED,
             'write_optimized_marker_layout': True, 'marker_layout': {'basename': DERIVED, 'fname': DERIVED},
             'stagei_basename': DERIVED, 'stagei_fname': DERIVED, 'stageii_fname': DERIVED, 'log_fname': DERIVED},
    'opt_settings': {'weights_type': DERIVED, 'weights': DERIVED, 'maxiter': 100, 'stagei_lr': 1e-3,
                     'extra_initial_rigid_adjustment': False},
    'opt_weights': {
        'smplh': dict(_OPT_WEIGHTS_SMPLX),
        'smplx': dict(_OPT_WEIGHTS_SMPLX),
        'smplx_grab_vtemplate': dict(
            stagei_wt_surf=10000.0, stagei_wt_init_hand=347.36, stagei_wt_init_finger=789.47, stagei_wt_init_finger_left=789.47,
            stagei_wt_init_finger_right=789.47, stagei_wt_init_head=220.69, stagei_wt_init_face=1100., stagei_wt_poseH=5.31,
            stagei_wt_poseF=28.97, stagei_wt_expr=6.99, stagei_wt_pose=3.00, stagei_wt_poseB=3.00, stagei_wt_betas=10.00,
            stagei_wt_init=300.00, stagei_wt_data=75.00, stagei_wt_annealing=[1., .5, .25, .125], stageii_wt_data=400,
            stageii_wt_velo=2.5, stageii_wt_dmpl=1.0, stageii_wt_expr=0.9, stageii_wt_poseB=1.6, stageii_wt_poseH=0.4,
            stageii_wt_poseF=15.0, stageii_wt_annealing=2.5),
    },
    'runtime': {'stagei_only': False},
}


class MissingMandatoryValue(ValueError):
    """A value the yaml marks ``???`` was not given (omegaconf raises its error of the same name)."""


def rm_spaces(s: str) -> str:
    """tools/run_tools.py: blanks removed from names taken from the capture path."""
    return s.replace(' ', '')


def resolve_gender(mocap_fname: str, fall_back_gender: str = 'error', subject_name=None, multi_subject: bool = False) -> str:
    """``resolve_mosh_subject_gender`` (tools/run_tools.py:88-122): ``settings.json`` next to the capture holds
    ``{"gender": ...}`` for one subject, ``{"<subject name>": {"gender": ...}}`` for several."""
    import json
    import os
    if multi_subject and subject_name is None:
        raise ValueError('For multi subject gender resolving the mocap.subject_name should be specified.')
    gender_fname = os.path.join(os.path.dirname(mocap_fname), 'settings.json')
    data = {}
    if os.path.exists(gender_fname):
        with open(gender_fname) as f:
            data = json.load(f)
    if multi_subject or (subject_name != 'null' and subject_name is not None):
        gender = data.get(subject_name, {}).get('gender', None)
    else:
        gender = data.get('gender', None)
    if gender is None:
        if fall_back_gender == 'error':
            raise FileNotFoundError(f'The gender of subject "{subject_name}" could not be determined from the settings file '
                                    f'{gender_fname}' if multi_subject else f'gender settings not found {gender_fname}')
        return fall_back_gender
    return gender


def _set_dotted(tree: dict, key: str, value, given: set):
    node = tree
    parts = key.split('.')
    for q in parts[:-1]:
        if not isinstance(node.get(q), dict):
            node[q] = {}
        node = node[q]
    node[parts[-1]] = value
    given.add(key)


def _merge(tree: dict, over: dict, given: set, prefix: str = ''):
    """Recursive merge of ``over`` into ``tree``; ``given`` collects the dotted keys the caller set."""
    for k, v in over.items():
        key = f'{prefix}{k}'
        if isinstance(v, dict) and isinstance(tree.get(k), dict):
            _merge(tree[k], v, given, key + '.')
        else:
            tree[k] = copy.deepcopy(v)
            given.add(key)
            if isinstance(v, dict):     # a whole subtree given: every leaf under it counts as given
                stack = [(key, v)]
                while stack:
                    p, d = stack.pop()
                    for kk, vv in d.items():
                        given.add(f'{p}.{kk}')
                        if isinstance(vv, dict):
                            stack.append((f'{p}.{kk}', vv))


def _parse_scalar(v):
    """The value of an ``a.b=v`` dotlist entry, as omegaconf's YAML parse of ``v`` would give it for plain scalars."""
    if not isinstance(v, str):
        return v
    low = v.strip().lower()
    if low in ('null', '~', ''):
        return None
    if low in ('true', 'false'):
        return low == 'true'
    for cast in (int, float):
        try:
            return cast(v)
        except ValueError:
            pass
    return v


def prepare_cfg(dict_cfg=None, **kwargs) -> AttrDict:
    """``MoSh.prepare_cfg`` (mosh_head.py:544-559) without omegaconf: the defaults of moshpp_conf.yaml, then the ``a.b=v``
    keyword overrides, then ``dict_cfg`` (a nested mapping), then every interpolation of the yaml computed from
    the merged values -- except where the caller set the value explicitly, which wins (as an explicit value replaces the
    interpolation in omegaconf).  ``mocap.fname``, ``dirs.work_base_dir`` and ``dirs.support_base_dir`` are required."""
    tree = copy.deepcopy(MOSHPP_CONF)
    given: set = set()
    for k, v in kwargs.items():                                     # keyword dotlist (mosh_head.py:554-555)
        _set_dotted(tree, k, _parse_scalar(v) if isinstance(v, str) else copy.deepcopy(v), given)
    if dict_cfg:
        _merge(tree, to_container(dict_cfg), given)
    for key in ('mocap.fname', 'dirs.work_base_dir', 'dirs.support_base_dir'):
        node = tree
        for q in key.split('.'):
            node = node[q]
        if node in (MISSING, None):
            raise MissingMandatoryValue(f'Missing mandatory value: {key}')

    mc, sm, mp, dr, opt = tree['mocap'], tree['surface_model'], tree['moshpp'], tree['dirs'], tree['opt_settings']

    def derive(key, fn):
        if key in given:
            return
        node = tree
        parts = key.split('.')
        for q in parts[:-1]:
            node = node[q]
        node[parts[-1]] = fn()

    fname = str(mc['fname'])
    derive('mocap.ds_name', lambda: rm_spaces(fname.split('/')[-3]))
    derive('mocap.session_name', lambda: rm_spaces(fname.split('/')[-2]))
    derive('mocap.basename', lambda: rm_spaces('.'.join(fname.split('/')[-1].split('.')[:-1])))

    def subject_names():
        from .mocap_interface import MocapSession
        return MocapSession(fname, 'mm').subject_names
    derive('mocap.subject_names', subject_names)
    sid = int(mc['subject_id'])
    derive('mocap.subject_name', lambda: mc['subject_names'][sid] if sid >= 0 else None)
    derive('mocap.multi_subject', lambda: len(mc['subject_names']) > 1 and sid >= 0)
    derive('surface_model.gender', lambda: resolve_gender(fname, 'error', mc['subject_name'], mc['multi_subject']))
    support, work, st = dr['support_base_dir'], dr['work_base_dir'], sm['type']
    derive('surface_model.fname', lambda: f"{support}/{st}/{sm['gender']}/model.pkl")
    derive('surface_model.dmpl_fname', lambda: f"{support}/{st}/{sm['gender']}/dmpl.pkl")
    derive('moshpp.head_marker_corr_fname', lambda: f'{support}/ssm_head_marker_corr.npz')
    derive('moshpp.pose_body_prior_fname', lambda: f'{support}/{st}/pose_body_prior.pkl')
    derive('moshpp.pose_hand_prior_fname', lambda: f'{support}/{st}/pose_hand_prior.npz')
    perseq = bool(mp['perseq_mosh_stagei'])
    derive('moshpp.stagei_frame_picker.stagei_mocap_fnames', lambda: [mc['fname']] if perseq else None)
    derive('dirs.session_subject_subfolders',
           lambda: f"{mc['session_name']}/{mc['subject_name']}" if mc['multi_subject'] else mc['session_name'])
    ds, ssf = mc['ds_name'], dr['session_subject_subfolders']
    derive('dirs.marker_layout.basename', lambda: f"{mc['basename']}_{st}" if perseq else f'{ds}_{st}')
    mlb = dr['marker_layout']['basename']
    derive('dirs.marker_layout.fname', lambda: f'{work}/{ds}/{ssf}/{mlb}.json' if perseq else f'{work}/{ds}/{mlb}.json')
    derive('dirs.stagei_basename', lambda: f"{mc['basename']}_{sm['gender']}" if perseq else sm['gender'])
    derive('dirs.stagei_fname', lambda: f"{work}/{ds}/{ssf}/{dr['stagei_basename']}_stagei.pkl")
    derive('dirs.stageii_fname', lambda: f"{work}/{ds}/{ssf}/{mc['basename']}_stageii.pkl")
    derive('dirs.log_fname', lambda: f"{work}/{ds}/{ssf}/{mc['basename']}.log")
    derive('opt_settings.weights_type', lambda: st)

    def weights():
        wt = opt['weights_type']
        if wt not in tree['opt_weights']:
            raise KeyError(f"opt_weights has no block for opt_settings.weights_type {wt!r} "
                           f"(the yaml has {sorted(tree['opt_weights'])}); set opt_settings.weights")
        return copy.deepcopy(tree['opt_weights'][wt])
    derive('opt_settings.weights', weights)
    return AttrDict.wrap(tree)


def to_container(cfg):
    """Plain nested dicts and lists of a configuration (``OmegaConf.to_container(cfg, resolve=True)``)."""
    if isinstance(cfg, dict) or (hasattr(cfg, 'keys') and hasattr(cfg, '__getitem__')):
        return {str(k): to_container(cfg[k]) for k in cfg.keys()}
    if isinstance(cfg, (list, tuple)):
        return [to_container(v) for v in cfg]
    return cfg
