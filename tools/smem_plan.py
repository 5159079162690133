"""Development tool (CPU): the workspace plan of a Stage-II job for synthetic configurations -- the library's own
plan_workspace (mosh2_host.h), through the test-only host build: shared-memory bytes per block, whether A, its factor and the
build scratch go to the per-block global workspace, and how large that is.
Usage: python tools/smem_plan.py [C1 C2 ... | CF80]   (CF80: CF with the reference's 80 expression coefficients)"""
import ctypes as C
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from moshpp_b200 import build, chmosh, lib, synth  # noqa: E402


def main():
    fn = C.CDLL(build.build_emu()).mosh2_emu_plan
    fn.argtypes = [C.POINTER(lib.ModelDesc), C.c_int32, C.c_int32, C.POINTER(C.c_int64)]
    fn.restype = C.c_int32
    d = tempfile.mkdtemp(prefix='mosh_plan_')
    for name in (sys.argv[1:] or ['C1', 'C2', 'C3', 'C4', 'CF', 'CH', 'CF80']):
        kw = dict(synth.REFERENCE_FACE) if name == 'CF80' else {}
        case = synth.make_case(d, 'CF' if name == 'CF80' else name, frames=2, write_mocap=False, **kw)
        pk, _, _ = chmosh.prepare_stageii(case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'], case['marker_meta'])
        h = lib.DescHolder(pk)
        print(name, 'markers', pk.n_markers, 'n1', len(pk.free_step1), 'n2', len(pk.free_step2), 'linear', pk.n_dmpl, flush=True)
        for prec, pname in ((lib.MOSH2_F32, 'f32'), (lib.MOSH2_F64, 'f64')):
            out = (C.c_int64 * 5)()
            assert fn(C.byref(h.desc), prec, 0, out) == 0
            fits = 'fits' if out[0] <= out[4] else 'DOES NOT FIT'
            print(f'  {pname}: shared {out[0]} B of {out[4]} ({fits}), '
                  f'{"global workspace " + str(out[1]) + " B per block" if out[2] else "workspace in shared memory"}, '
                  f'{out[3]}-marker tiles')


if __name__ == '__main__':
    main()
