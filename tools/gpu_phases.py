"""Development tool: phase clock breakdown of the Stage-II kernel (needs moshpp_b200/libmosh2_prof.so, built by
``python -m moshpp_b200.build --profile``).

Usage: python tools/gpu_phases.py C2 [frames] [L:W | product] [f32|f64]

``product``: the schedule the product plans for the sequence (chmosh.plan_chunk_len with the default warm-up, its fully
solved part and the first chunk's extra frames); ``python tools/gpu_phases.py C5 4000 product`` is the launch bench.py
times.  The clocks are those of the first launch (all chunks); with the product schedule the verified launch
(boundary check and repair rounds) is timed after it, launch by launch."""
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from moshpp_b200 import chmosh, lib, synth  # noqa: E402
from moshpp_b200.mocap_interface import MocapSession  # noqa: E402

NAMES = ['ev.fullpose', 'ev.rodrigues', 'ev.fk||blend', 'ev.skin+prior', 'ev.markers', 'ev.reduce', 'bd.pre', 'bd.T1',
         'bd.T2', 'bd.T3', 'bd.closed', 'gn.init', 'gn.w0 panel+update', 'gn.w0 diag block', 'gn.w0 barrier wait', 'gn.solves', 'minimize(all)',
         'chunk(all)', 'ev.fk alone', 'ev.prior alone', 'sf.stage_setup', 'sf.accept logic', 'sf.symv+reduce (pre GN)', 'sf.step+symv (post GN)', 'sf.output', 'sf.other']


def gpu_name():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def main():
    name = sys.argv[1] if len(sys.argv) > 1 else 'C2'
    frames = int(sys.argv[2]) if len(sys.argv) > 2 else 16
    sched = sys.argv[3] if len(sys.argv) > 3 else '0:0'
    prec = lib.MOSH2_F64 if (len(sys.argv) > 4 and sys.argv[4] == 'f64') else lib.MOSH2_F32
    d = tempfile.mkdtemp(prefix='mosh_phase_')
    case = synth.make_case(d, name, frames=frames)
    pk, opts, _ = chmosh.prepare_stageii(case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])
    mocap = MocapSession(case['mocap_fname'], 'mm')
    obs, vis = mocap.frames_for_labels(case['latent_labels'], range(len(mocap)))
    path = os.path.join(ROOT, 'moshpp_b200', os.environ.get('MOSH2_PROF_LIB', 'libmosh2_prof.so'))
    model = lib.Model(pk, device=0, library_path=path)
    F = obs.shape[0]
    if sched == 'product':
        W, WF = chmosh.DEFAULT_WARMUP, chmosh.DEFAULT_WARMUP_FULL
        extra = chmosh.first_chunk_extra(W, WF)
        L = chmosh.plan_chunk_len([F], chmosh.NUM_SMS, W, WF, first_extra=extra)
        job = model.job(F, opts, chunk_len=L, chunk_warmup=W, warmup_full=WF, precision=prec, first_extra=extra)
    else:
        L, W = (int(x) for x in sched.split(':'))
        WF, extra = -1, 0
        job = model.job(F, opts, chunk_len=L, chunk_warmup=W, precision=prec)
    job.upload(obs, vis)
    job.launch(); job.sync()
    job.launch(); job.sync()
    ms = job.kernel_ms()
    tot = job.totals()
    clk = np.zeros(32, dtype=np.int64)
    model.lib.mosh2_dev_phase_clocks.argtypes = [C.c_void_p, C.POINTER(C.c_longlong)]
    model.lib.mosh2_dev_phase_clocks(job.handle, clk.ctypes.data_as(C.POINTER(C.c_longlong)))
    info = dict(gpu=gpu_name(), config=name, frames=F, chunk_len=L, chunk_warmup=W, warmup_full=WF, first_extra=extra,
                kernel_ms=ms, totals=tot, chunks=job.num_chunks)
    if sched == 'product':
        verified = []
        for _ in range(3):
            _, rep = chmosh.launch_verified(job, chmosh.BOUNDARY_TOL['fast'])
            verified.append(rep['kernel_ms'])
        info['verified_kernel_ms'] = verified        # [first launch, repair rounds...] per pass (profiled build)
    print(json.dumps(info))
    nb = max(1, tot['builds'])
    chunk = clk[17]
    for i, n in enumerate(NAMES):
        print(f'{n:16s} {clk[i]/nb:10.0f} cycles/build  {100*clk[i]/max(1,chunk):5.1f}% of chunk time')


if __name__ == '__main__':
    main()
