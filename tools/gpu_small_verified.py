"""Development tool (GPU): a small chunked + verified + repaired solve."""
import os, sys, tempfile
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from moshpp_b200 import chmosh, lib, synth
from moshpp_b200.mocap_interface import MocapSession
for name, prec in (('C2', lib.MOSH2_F32), ('C3', lib.MOSH2_F32), ('C4', lib.MOSH2_F64)):
    case = synth.make_case(tempfile.mkdtemp(), name, frames=40, n_verts=None if name == 'C4' else 1500)
    pk, opts, _ = chmosh.prepare_stageii(case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])
    mocap = MocapSession(case['mocap_fname'], 'mm')
    obs, vis = mocap.frames_for_labels(case['latent_labels'], range(len(mocap)))
    model = lib.Model(pk, device=0)
    seq = model.solve(obs, vis, opts, precision=prec)
    job = model.job([25, 15], opts, chunk_len=4, chunk_warmup=6, warmup_full=3, precision=prec)     # a batch job of two sequences
    res, rep = chmosh.solve_verified(job, obs, vis, tol=(1e-7, 1e-7, 1e-8, 1e-7), max_rounds=8)
    print(name, 'rounds', rep['rounds'], 'repaired', rep['repaired_chunks'], 'delta first', np.round(rep['boundary_delta_first'], 5),
          'last', rep['boundary_delta_max'], '| vs sequential (first sequence)', np.abs(res.pose[:25] - seq.pose[:25]).max())
    job.close(); model.close()
lib.load_library().mosh2_release_cached_memory()
print('OK')
