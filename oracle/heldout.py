"""Held-out marker validation of Stage II (DESIGN.md section 12) on the float64 oracle.

A fold is a set of latent labels.  Its solve is the unchanged ``stageii.StageIISolver`` frame loop on the capture with every sample
of the fold's markers deleted: the markers stay in the layout and are visible in no frame, so the visibility count, the data
weight and the annealing are those of a capture that never saw them, and a frame left without a visible marker is skipped.  The
error of a held-out marker i in a frame t the fold processed, where the capture observes i, is |sim_i - obs_i| in metres, sim_i
the marker simulated on the fold's solved body through the Stage-I attachment; everywhere else it is NaN.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np

from .stageii import StageIISolver, frames_from_mocap


def heldout_errors(mocap_fname, cfg, markers_latent, latent_labels, betas, marker_meta, folds: Sequence[Sequence[str]], *,
                   mocap=None, robust_data_sigma: Optional[float] = None) -> dict:
    """The sequential fold solves of ``folds`` (lists of latent labels) on the capture ``mocap_fname`` (or ``mocap``, as
    ``stageii.mosh_stageii`` takes it).  Returns err [n_folds, F, K] (metres; F the selected frames, K the largest fold, entry
    (k, t, r) for the r-th marker of fold k in latent order, NaN where undefined), and per fold the Jacobian builds of its solve
    (``j_evals``) and the frames it processed (``frame_ids``)."""
    if mocap is None:
        from moshpp_b200.mocap_interface import MocapSession
        mocap = MocapSession(mocap_fname, mocap_unit=cfg.mocap.unit, mocap_rotate=cfg.mocap.rotate,
                             only_subjects=[cfg.mocap.subject_name] if cfg.mocap.multi_subject else None)
    n = len(mocap.markers)
    sel = list(range(cfg.mocap.start_fidx, n if cfg.mocap.end_fidx == -1 else cfg.mocap.end_fidx, cfg.mocap.ds_rate))
    markers = np.array(mocap.markers[sel], dtype=np.float64)
    latent = list(latent_labels)
    full = frames_from_mocap(markers, mocap.labels, latent)
    idx = [sorted({latent.index(l) for l in fold}) for fold in folds]
    err = np.full((len(folds), len(sel), max(len(f) for f in idx)), np.nan)
    j_evals, frame_ids = [], []
    for k, fold in enumerate(idx):
        hidden = {latent[i] for i in fold}
        masked = markers.copy()
        masked[:, [c for c, l in enumerate(mocap.labels) if l in hidden]] = np.nan        # deleted samples: missing in every frame
        solver = StageIISolver(cfg, markers_latent, latent, betas, marker_meta, robust_data_sigma=robust_data_sigma)
        sims = {}
        solver.solve_range(frames_from_mocap(masked, mocap.labels, solver.latent_labels),
                           on_frame=lambda fi: sims.__setitem__(fi, solver.evaluate(False)['markers'].copy()))
        for t, sim in sims.items():
            vis_t, obs_t = full[t]
            for r, i in enumerate(fold):
                hit = np.flatnonzero(vis_t == i)
                if len(hit):
                    err[k, t, r] = np.linalg.norm(sim[i] - obs_t[hit[0]])
        j_evals.append(int(solver.stats['j_evals']))
        frame_ids.append(np.array(sorted(sims)))
    return dict(err=err, j_evals=np.array(j_evals), frame_ids=frame_ids)
