"""Stage-I frame picker: which capture frames Stage I fits (the reference's ``frame_picker.py:43-213``).

Each picker returns ``(frames, fnames)``: an object array of per-frame ``{label: xyz}`` dictionaries (the available samples
of the frame, metres) and the matching array of keys ``<capture path>_<number:06d>``.  Given the same state of numpy's
global legacy RNG the picks equal the reference's: the same ``np.random`` calls are made in the same order, quirks included
(SURVEY.md Appendix B-14):

* ``random``: every capture draws ``np.random.choice(len(mocap), num_frames)`` WITH replacement, before any seeding; the key
  numbers the draw, not the file frame; captures are read until more than 100 keys exist; a frame qualifies when its
  available labels without a ``*`` reach ``least_avail_markers`` times its available labels; too few frames lower the
  threshold by 0.01 and start again, and that call drops ``exclude_markers``;
* ``random_strict``: reseeds on entry; skips captures that could not be read (``read_status``); a frame's availability is
  ``marker_availability_mask`` over ALL the capture's columns; raises ``ValueError`` when fewer than ``num_frames`` qualify;
* ``manual``: entries ``<capture path>_<frame id>``.
"""
from __future__ import annotations

import os
from typing import Dict, List

import numpy as np

from .mocap_interface import MocapSession


def _frame_dict(mocap: MocapSession, t: int, ok: np.ndarray) -> Dict[str, np.ndarray]:
    """Frame ``t`` of ``MocapSession.markers_asdict()`` (``ok``: the availability mask of the capture)."""
    return {l: mocap.markers[t, c] for c, l in enumerate(mocap.labels) if ok[t, c]}


def _session(fname, mocap_unit, mocap_rotate, only_subjects, only_markers, exclude_markers, labels_map) -> MocapSession:
    return MocapSession(mocap_fname=fname, mocap_unit=mocap_unit, mocap_rotate=mocap_rotate, only_subjects=only_subjects,
                        only_markers=only_markers, exclude_markers=exclude_markers, labels_map=labels_map)


def load_marker_sessions_manual(mocap_fnames: List[str], mocap_unit: str, mocap_rotate: list = None, only_subjects: List[str] = None,
                                only_markers=None, exclude_markers=None, labels_map={}):
    """The listed frames: entries ``/path/to/capture.ext_<frame id>`` (split at the last ``_``)."""
    frames, keys = [], []
    for entry in mocap_fnames:
        path, _, frame_id = entry.rpartition('_')
        t = int(frame_id)
        if not os.path.exists(path):                            # (an assertion in the reference)
            raise AssertionError(FileNotFoundError(path))
        keys.append(f'{path}_{t:06d}')
        m = _session(path, mocap_unit, mocap_rotate, only_subjects, only_markers, exclude_markers, labels_map)
        frames.append(_frame_dict(m, t, MocapSession.marker_availability_mask(m.markers)))
    return np.array(frames), np.array(keys)


def load_marker_sessions_random(mocap_fnames: List[str], mocap_unit: str, mocap_rotate: list = None, num_frames: int = 12,
                                only_subjects: List[str] = None, seed: int = None, least_avail_markers: float = .1,
                                only_markers=None, exclude_markers=None, labels_map={}):
    """``num_frames`` frames drawn at random from the captures; see the module docstring for the rules."""
    drawn: Dict[str, dict] = {}
    for fname in mocap_fnames:
        m = _session(fname, mocap_unit, mocap_rotate, only_subjects, only_markers, exclude_markers, labels_map)
        ok = MocapSession.marker_availability_mask(m.markers)
        for i, t in enumerate(np.random.choice(len(m), num_frames)):
            drawn[f'{fname}_{i:06d}'] = _frame_dict(m, int(t), ok)
        if len(drawn) > 100:
            break
    order = list(range(len(drawn)))
    if seed is not None:
        np.random.seed(seed=seed)
    np.random.shuffle(order)
    keys, dicts = list(drawn.keys()), list(drawn.values())
    frames, names = [], []
    for j in order:
        d = dicts[j]
        counted = sum(1 for label, xyz in d.items() if '*' not in label and not np.isnan(xyz).any())
        if counted >= least_avail_markers * len(d):
            frames.append(d)
            names.append(keys[j])
        if len(frames) >= num_frames:
            break
    if len(frames) < num_frames:
        lowered = least_avail_markers - 0.01
        if lowered < 0.01:
            raise ValueError(f'fewer than {num_frames} frames have {lowered * 100.:.1f}% of their markers available')
        return load_marker_sessions_random(mocap_fnames, mocap_unit=mocap_unit, mocap_rotate=mocap_rotate, seed=seed,
                                           num_frames=num_frames, only_subjects=only_subjects, least_avail_markers=lowered,
                                           only_markers=only_markers, labels_map=labels_map)     # (exclude_markers dropped)
    return np.array(frames), np.array(names)


def load_marker_sessions_random_strict(mocap_fnames: List[str], mocap_unit: str, mocap_rotate: list = None, num_frames: int = 12,
                                       only_subjects: List[str] = None, seed: int = None, least_avail_markers: float = .1,
                                       only_markers=None, exclude_markers=None, labels_map={}):
    """``num_frames`` frames drawn at random among those with at least ``least_avail_markers`` of the capture's columns
    available; the threshold is never lowered."""
    np.random.seed(seed=seed)
    if not 0.1 <= least_avail_markers <= 1.0:                   # (an assertion in the reference)
        raise AssertionError(f'least_avail_markers {least_avail_markers} outside [0.1, 1.0]')
    qualified: Dict[str, dict] = {}
    for fname in mocap_fnames:
        m = _session(fname, mocap_unit, mocap_rotate, only_subjects, only_markers, exclude_markers, labels_map)
        if not m.read_status:
            continue
        ok = MocapSession.marker_availability_mask(m.markers)
        share = ok.sum(-1) / ok.shape[1]
        taken = 0
        for t in np.random.choice(len(m), len(m), replace=False):
            if share[t] >= least_avail_markers:
                qualified[f'{fname}_{t:06d}'] = _frame_dict(m, int(t), ok)
                taken += 1
            if taken >= num_frames:
                break
        if len(qualified) > 100:
            break
    if len(qualified) < num_frames:
        raise ValueError(f'fewer than {num_frames} frames have {least_avail_markers * 100.:.1f}% of the markers available: use '
                         'moshpp.stagei_frame_picker.type random, or a lower moshpp.stagei_frame_picker.least_avail_markers '
                         '(0.1 to 1.0)')
    ids = np.random.choice(len(qualified), num_frames, replace=False)
    return np.array(list(qualified.values()))[ids], np.array(list(qualified.keys()))[ids]
