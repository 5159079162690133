"""The MoSh++ head without the reference: ``MoSh`` and ``run_moshpp_once`` (src/moshpp/mosh_head.py:65-301,561-606), plus
``run_moshpp_subject``, which solves all captures of a subject in one launch, and for a dataset the reference's jobs filter
(``universal_mosh_jobs_filter``, tools/run_tools.py:45-67) and ``run_moshpp_jobs``, which solves the captures of many subjects
in one launch per group of kernel-compatible subjects.

The reference's head imports human_body_prior, loguru, omegaconf, psbody and the marker-layout tools, so the plug-in point
of its two stage functions cannot be imported where psbody is absent.  This one runs on the package alone:

* configuration: ``cfg.prepare_cfg`` (moshpp_conf.yaml and its resolvers as plain functions), stored as plain dicts;
* Stage-I frames: ``frame_picker`` (the reference's pickers, same picks for the same RNG state);
* stages: ``stagei.mosh_stagei`` and ``chmosh.mosh_stageii`` by default, or any callables of the same signatures;
* results: the reference's pickle files at the reference's paths (``dirs.stagei_fname`` / ``dirs.stageii_fname``), read back
  as caches on the next run; ``amass_io`` for the Stage-II merge and the AMASS npz.

Logging goes through the ``logging`` logger ``moshpp_b200`` (loguru is absent); the head adds no handlers.  A marker layout
that does not exist is not created (the reference derives it from its label-to-vertex tables): the head raises
``FileNotFoundError`` instead.
"""
from __future__ import annotations

import copy
import glob
import logging
import os
import pickle
import time
from typing import List, Optional, Union

import numpy as np

from . import amass_io
from . import frame_picker
from .cfg import prepare_cfg, to_container

logger = logging.getLogger('moshpp_b200')


def _dump(obj, fname: str):
    os.makedirs(os.path.dirname(os.path.abspath(fname)), exist_ok=True)
    with open(fname, 'wb') as f:
        pickle.dump(obj, f)


def _load(fname: str):
    with open(fname, 'rb') as f:
        return pickle.load(f)


class MoSh:
    """mosh_head.py:65-301: configuration, Stage-I frame choice, and the two stages with their pickle caches."""

    def __init__(self, dict_cfg=None, **kwargs) -> None:
        self.cfg = prepare_cfg(dict_cfg=dict_cfg, **kwargs)
        mc = self.cfg.mocap
        if mc.multi_subject:
            logger.info('MoCap is multi subject. Available subjects (id:name): %s', dict(enumerate(mc.subject_names)))
            logger.info('mocap.subject_id: %s is selected: %s', mc.subject_id, mc.subject_name)
        self.stagei_fname = self.cfg.dirs.stagei_fname
        self.stageii_fname = self.cfg.dirs.stageii_fname
        self.stagei_data = None
        self.stageii_data = None
        if self.cfg.moshpp.verbosity < 0:           # a status call (mosh_head.py:93)
            return
        logger.info('mocap_fname: %s; stagei_fname: %s; stageii_fname: %s', mc.fname, self.stagei_fname, self.stageii_fname)
        if not os.path.exists(self.cfg.surface_model.fname):
            raise AssertionError(FileNotFoundError(f'surface_model_fname not found: {self.cfg.surface_model.fname}'))
        if self.cfg.dirs.marker_layout.fname is None:                                             # mosh_head.py:120-122
            self.cfg.dirs.marker_layout.fname = os.path.join(os.path.dirname(os.path.dirname(mc.fname)),
                                                             f'{self.cfg.surface_model.type}_{mc.ds_name}.json')

    def _only_subjects(self):
        return [self.cfg.mocap.subject_name] if self.cfg.mocap.multi_subject else None

    def prepare_stagei_frames(self, stagei_mocap_fnames: List[str] = None):
        """mosh_head.py:135-198: without ``stagei_mocap_fnames`` the captures come from the capture's directory (same
        extension); of more than ``num_frames`` captures, ``num_frames`` are drawn without replacement."""
        from .mocap_interface import general_labels_map
        fp = self.cfg.moshpp.stagei_frame_picker
        if stagei_mocap_fnames is None:
            if fp.type == 'manual':
                raise AssertionError(ValueError('with frame_picker.type manual you should provide list of [/path/to/mocap.c3d_frameid]'))
            ext = os.path.basename(self.cfg.mocap.fname).split('.')[-1]
            mocap_fnames = sorted(glob.glob(os.path.join(os.path.dirname(self.cfg.mocap.fname), f'*.{ext}')))
            assert len(mocap_fnames) > 0
            mc_ids = np.random.choice(len(mocap_fnames), fp.num_frames, replace=False) if len(mocap_fnames) > fp.num_frames \
                else np.arange(len(mocap_fnames))
            stagei_mocap_fnames = [mocap_fnames[i] for i in mc_ids]
            logger.debug('%d subject specific mocap(s) are selected for mosh stagei.', len(stagei_mocap_fnames))
        mc = self.cfg.mocap
        common = dict(mocap_unit=mc.unit, mocap_rotate=mc.rotate, only_markers=mc.only_markers, only_subjects=self._only_subjects(),
                      exclude_markers=mc.exclude_markers, labels_map=general_labels_map())
        if fp.type == 'random':
            frames, fnames = frame_picker.load_marker_sessions_random(stagei_mocap_fnames, num_frames=fp.num_frames, seed=fp.seed,
                                                                      least_avail_markers=fp.least_avail_markers, **common)
        elif fp.type == 'random_strict':
            frames, fnames = frame_picker.load_marker_sessions_random_strict(stagei_mocap_fnames, num_frames=fp.num_frames, seed=fp.seed,
                                                                             least_avail_markers=fp.least_avail_markers, **common)
        elif fp.type == 'manual':
            frames, fnames = frame_picker.load_marker_sessions_manual(stagei_mocap_fnames, **common)
        else:
            raise ValueError(f'Wrong frame_picker value: {fp.type}')
        logger.debug('Using frames for stage-i: %s', fnames)
        return frames, fnames

    def mosh_stagei(self, mosh_stagei_func=None):
        """mosh_head.py:200-266.  ``mosh_stagei_func`` defaults to ``stagei.mosh_stagei``."""
        if os.path.exists(self.stagei_fname):
            self.stagei_data = _load(self.stagei_fname)
            prev = self.stagei_data['stagei_debug_details']['cfg']['surface_model']['fname']
            if prev != self.cfg.surface_model.fname:
                raise AssertionError(ValueError(f'The surface_model_fname used for previous stagei ({prev}) is different than the '
                                                f'current surface model ({self.cfg.surface_model.fname})'))
            logger.info('loading mosh stagei results from %s', self.stagei_fname)
            return self.stagei_fname
        if mosh_stagei_func is None:
            from .stagei import mosh_stagei as mosh_stagei_func
        stagei_frames, stagei_fnames = self.prepare_stagei_frames(self.cfg.moshpp.stagei_frame_picker.stagei_mocap_fnames)
        layout = self.cfg.dirs.marker_layout.fname
        if not os.path.exists(layout):
            raise FileNotFoundError(f'marker layout {layout} does not exist.  The reference creates a missing layout from the '
                                    'labels of the picked frames and its own label-to-vertex tables, which are not part of this '
                                    'package: write the layout json (e.g. with stagei.write_marker_layout) or set '
                                    'dirs.marker_layout.fname')
        logger.info('Attempting mosh stagei to create %s', self.stagei_fname)
        tm = time.time()
        stagei_data = mosh_stagei_func(stagei_frames=stagei_frames, cfg=self.cfg, betas_fname=self.cfg.moshpp.betas_fname,
                                       v_template_fname=self.cfg.moshpp.v_template_fname)
        dbg = stagei_data['stagei_debug_details']
        dbg['stagei_fnames'] = stagei_fnames
        dbg['stagei_frames'] = stagei_frames
        dbg['cfg'] = to_container(self.cfg)
        dbg['stagei_elapsed_time'] = time.time() - tm
        _dump(stagei_data, self.stagei_fname)
        logger.debug('created stagei_fname: %s', self.stagei_fname)
        self.stagei_data = stagei_data
        if self.cfg.dirs.write_optimized_marker_layout:
            MoSh.dump_stagei_marker_layout(self.stagei_fname)
        return self.stagei_fname

    def _stageii_args(self):
        if self.stagei_data is None:
            raise ValueError(f'stagei_fname results could not be found: {self.stagei_fname}. please run stagei first.')
        d = self.stagei_data
        return dict(markers_latent=d['markers_latent'], latent_labels=d['latent_labels'], betas=d['betas'],
                    marker_meta=d['marker_meta'], v_template_fname=d.get('v_template_fname'))

    def mosh_stageii(self, mosh_stageii_func=None):
        """mosh_head.py:268-301.  ``mosh_stageii_func`` defaults to ``chmosh.mosh_stageii``."""
        args = self._stageii_args()
        if os.path.exists(self.stageii_fname):
            self.stageii_data = _load(self.stageii_fname)
            logger.info('loading mosh stageii results from %s', self.stageii_fname)
            return self.stageii_fname
        if mosh_stageii_func is None:
            from .chmosh import mosh_stageii as mosh_stageii_func
        logger.info('attempting mosh stageii to create %s', self.stageii_fname)
        tm = time.time()
        stageii_data = mosh_stageii_func(mocap_fname=self.cfg.mocap.fname, cfg=self.cfg, **args)
        self.stageii_data = amass_io.merge_stageii(stageii_data, self.stagei_data, to_container(self.cfg), time.time() - tm,
                                                   self.stageii_fname)
        logger.debug('created stageii_fname: %s', self.stageii_fname)
        return self.stageii_fname

    @staticmethod
    def extract_marker_layout_from_mosh(mosh_stagei_pkl_fname: Union[str, dict], template_marker_layout_fname: str = None) -> dict:
        """mosh_head.py:561-581: the layout of a Stage-I result with the optimised vertex ids."""
        mosh_stagei = mosh_stagei_pkl_fname if isinstance(mosh_stagei_pkl_fname, dict) else _load(mosh_stagei_pkl_fname)
        opt_marker_vids = mosh_stagei['markers_latent_vids']
        if template_marker_layout_fname:
            from .stagei import load_marker_layout
            marker_meta = load_marker_layout(template_marker_layout_fname)
        else:
            marker_meta = copy.deepcopy(mosh_stagei['marker_meta'])
        for l in marker_meta['marker_vids']:
            if l in opt_marker_vids:
                marker_meta['marker_vids'][l] = opt_marker_vids[l]
        return marker_meta

    @staticmethod
    def dump_stagei_marker_layout(mosh_stagei_pkl_fname: str, out_marker_layout_fname: str = None,
                                  template_marker_layout_fname: str = None) -> str:
        """mosh_head.py:303-340, the json only (the .ply / .c3d companions are viewer files)."""
        from .stagei import write_marker_layout
        if not mosh_stagei_pkl_fname.endswith('.pkl'):
            raise AssertionError(ValueError(f'mosh_stagei_pkl_fname should be a valid pkl file: {mosh_stagei_pkl_fname}'))
        marker_meta = MoSh.extract_marker_layout_from_mosh(mosh_stagei_pkl_fname, template_marker_layout_fname)
        if out_marker_layout_fname is None:
            out_marker_layout_fname = mosh_stagei_pkl_fname.replace('.pkl', '.json')
        write_marker_layout(out_marker_layout_fname, marker_meta)
        logger.info('created %s', out_marker_layout_fname)
        return out_marker_layout_fname

    @staticmethod
    def load_as_amass_npz(stageii_pkl_data_or_fname, stageii_npz_fname=None, stagei_npz_fname=None, include_markers: bool = False,
                          include_extra_details: bool = False) -> dict:
        """mosh_head.py:444-541 (``amass_io.load_as_amass_npz``)."""
        return amass_io.load_as_amass_npz(stageii_pkl_data_or_fname, stageii_npz_fname, stagei_npz_fname, include_markers,
                                          include_extra_details)


def _loss_line(errs) -> str:
    return ' | '.join(f'{k} = {np.sum(np.asarray(v) ** 2):2.2e}' for k, v in errs.items())


def run_moshpp_once(cfg, *, stagei_func=None, stageii_func=None) -> MoSh:
    """mosh_head.py:584-606: Stage I (or its cache), then Stage II (or its cache) unless ``runtime.stagei_only``.  ``cfg``: the
    keyword overrides of ``MoSh`` (dotted keys).  The stage functions default to ``stagei.mosh_stagei`` and
    ``chmosh.mosh_stageii``."""
    mp = MoSh(**cfg)
    mp.mosh_stagei(stagei_func)
    logger.debug('Final mosh stagei loss: %s', _loss_line(mp.stagei_data['stagei_debug_details']['stagei_errs']))
    if not mp.cfg.runtime.stagei_only:
        mp.mosh_stageii(stageii_func)
        logger.debug('Final mosh stageii loss: %s', _loss_line(mp.stageii_data['stageii_debug_details']['stageii_errs']))
    return mp


def run_moshpp_subject(cfg, mocap_fnames: Optional[List[str]] = None, *, stagei_func=None, stageii_batch_func=None) -> List[MoSh]:
    """All captures of one subject: Stage I once (through the same cache as ``MoSh``: the capture of ``cfg`` decides its
    path), then every capture without a Stage-II pickle in ONE ``chmosh.mosh_stageii_batch`` call (one launch on the GPU).
    Each capture's pickle is written at the path, and with the contents, that ``run_moshpp_once`` of that capture would
    produce; only the timing entries differ (``stageii_elapsed_time`` is the time of the whole batch).

    ``cfg``: the keyword overrides of ``MoSh`` (dotted keys) for one capture of the subject; ``mocap_fnames``: the captures
    (default: every file with the capture's extension in its directory).  Returns one ``MoSh`` per capture, its
    ``stageii_data`` set."""
    cfg = dict(cfg)
    head = MoSh(**cfg)
    if head.cfg.moshpp.perseq_mosh_stagei:
        raise ValueError('moshpp.perseq_mosh_stagei fits a shape per capture: run run_moshpp_once for each capture')
    if mocap_fnames is None:
        ext = os.path.basename(head.cfg.mocap.fname).split('.')[-1]
        mocap_fnames = sorted(glob.glob(os.path.join(os.path.dirname(head.cfg.mocap.fname), f'*.{ext}')))
    head.mosh_stagei(stagei_func)
    heads = []
    for fn in mocap_fnames:
        mp = MoSh(**dict(cfg, **{'mocap.fname': fn}))
        if mp.stagei_fname != head.stagei_fname:
            raise ValueError(f'{fn} belongs to another Stage I ({mp.stagei_fname}, not {head.stagei_fname})')
        mp.stagei_data = head.stagei_data
        heads.append(mp)
    if head.cfg.runtime.stagei_only:
        return heads
    todo = []
    for mp in heads:
        if os.path.exists(mp.stageii_fname):
            mp.stageii_data = _load(mp.stageii_fname)
            logger.info('loading mosh stageii results from %s', mp.stageii_fname)
        else:
            todo.append(mp)
    if not todo:
        return heads
    if stageii_batch_func is None:
        from .chmosh import mosh_stageii_batch as stageii_batch_func
    batch_cfg = todo[0].cfg
    logger.info('attempting mosh stageii of %d captures in one batch', len(todo))
    tm = time.time()
    results = stageii_batch_func(mocap_fnames=[mp.cfg.mocap.fname for mp in todo], cfg=batch_cfg, **head._stageii_args())
    elapsed = time.time() - tm
    for mp, data in zip(todo, results):
        for k in ('optimize_fingers', 'optimize_face'):         # the Stage-II gating the solver applied to its cfg
            mp.cfg.moshpp[k] = batch_cfg.moshpp[k]
        mp.stageii_data = amass_io.merge_stageii(data, head.stagei_data, to_container(mp.cfg), elapsed, mp.stageii_fname)
        logger.debug('created stageii_fname: %s', mp.stageii_fname)
    return heads


def universal_mosh_jobs_filter(total_jobs, only_stagei: bool = False, determine_shape_for_each_seq: bool = False) -> list:
    """tools/run_tools.py:45-67: the jobs (``MoSh`` keyword overrides, dotted keys) that still have work to do.  A job whose
    Stage-II pickle exists is done.  A job's key is ``<dataset>_<session>`` of its capture path (``_<capture file>`` added under
    ``moshpp.perseq_mosh_stagei``, ``_<session>_<subject>`` for a chosen subject of a multi-subject capture); the first job of a
    key whose Stage I does not exist yet is kept and, unless ``determine_shape_for_each_seq``, the later jobs of that key are
    dropped: one of them makes the shape the others need.  ``only_stagei``: jobs whose Stage I exists are dropped too."""
    filtered_jobs, exclude_keys = [], []
    for cur_job in total_jobs:
        mocap_fname_split = cur_job['mocap.fname'].split('/')
        mocap_key = '_'.join(mocap_fname_split[-3:-1])
        mosh_cfg = prepare_cfg(**copy.deepcopy(cur_job))
        if mosh_cfg.moshpp.perseq_mosh_stagei:
            mocap_key += f'_{mocap_fname_split[-1]}'
        if mosh_cfg.mocap.subject_id >= 0 and mosh_cfg.mocap.multi_subject:
            mocap_key += f'_{mosh_cfg.mocap.session_name}'
            mocap_key += f'_{mosh_cfg.mocap.subject_name}'
        if mocap_key in exclude_keys:
            continue
        if os.path.exists(mosh_cfg.dirs.stageii_fname):
            continue
        if not os.path.exists(mosh_cfg.dirs.stagei_fname) and not determine_shape_for_each_seq:
            exclude_keys.append(mocap_key)
        if only_stagei and os.path.exists(mosh_cfg.dirs.stagei_fname):
            continue
        filtered_jobs.append(cur_job)
    return filtered_jobs


def run_moshpp_jobs(jobs, *, stagei_func=None, stageii_subjects_func=None) -> List[MoSh]:
    """A dataset: ``run_moshpp_once`` of every job (``MoSh`` keyword overrides, dotted keys), with the Stage-II solves of all
    subjects in one ``chmosh.mosh_stageii_subjects`` call -- one launch per group of kernel-compatible subjects instead of one
    per subject or capture.

    The jobs are grouped by their Stage-I pickle (``dirs.stagei_fname``): one group per subject, or per capture under
    ``moshpp.perseq_mosh_stagei``.  Each group's Stage I is run (from its first job's configuration, as ``run_moshpp_once`` of
    that job would) or loaded through ``MoSh.mosh_stagei``.  Every job without a Stage-II pickle is then solved; its pickle
    is written at the path, and with the contents, that ``run_moshpp_once`` of that job produces, apart from the timing
    entries (``stageii_elapsed_time`` is the time of the whole call).  Returns one ``MoSh`` per job, in the order of ``jobs``."""
    heads = [MoSh(**dict(job)) for job in jobs]
    groups = {}
    for mp in heads:
        groups.setdefault(mp.stagei_fname, []).append(mp)
    subjects, members = [], []
    for group in groups.values():
        for mp in group:                        # (the first job makes the Stage I, the others load it)
            mp.mosh_stagei(stagei_func)
        if group[0].cfg.runtime.stagei_only:
            continue
        todo = []
        for mp in group:
            if os.path.exists(mp.stageii_fname):
                mp.stageii_data = _load(mp.stageii_fname)
                logger.info('loading mosh stageii results from %s', mp.stageii_fname)
            else:
                todo.append(mp)
        if todo:
            subjects.append(dict(cfg=todo[0].cfg, mocap_fnames=[mp.cfg.mocap.fname for mp in todo], **todo[0]._stageii_args()))
            members.append(todo)
    if not subjects:
        return heads
    if stageii_subjects_func is None:
        from .chmosh import mosh_stageii_subjects as stageii_subjects_func
    logger.info('attempting mosh stageii of %d captures of %d subjects', sum(len(t) for t in members), len(subjects))
    tm = time.time()
    results = stageii_subjects_func(subjects)
    elapsed = time.time() - tm
    for sub, todo, outs in zip(subjects, members, results):
        for mp, data in zip(todo, outs):
            for k in ('optimize_fingers', 'optimize_face'):     # the Stage-II gating the solver applied to its cfg
                mp.cfg.moshpp[k] = sub['cfg'].moshpp[k]
            mp.stageii_data = amass_io.merge_stageii(data, mp.stagei_data, to_container(mp.cfg), elapsed, mp.stageii_fname)
            logger.debug('created stageii_fname: %s', mp.stageii_fname)
    return heads
