"""The SMPL-X face path at the reference's size: 80 expression coefficients (moshpp_conf.yaml: betas_expr_start_id 300,
num_expressions 80, on a model file with 400 shape components), against float64.

The CF fixture fits 8 expressions, so its linear block is 10x narrower than in real use: Step 2 has n2 = 194 free variables
at 80 expressions against 122 at 8, and the float64 joint-direction tables (3 nJ nd words each: dtg and c_jd) grow to 106 KB
apiece.  This module covers that size:
  * the workspace plan (mosh2_host::plan_workspace, through the host build) of every configuration the reference's defaults
    produce, Stage II and the Stage-I packs, at the CF marker count and at a denser layout, in both precisions: every job
    must be possible (the exact preset runs float64);
  * on the host build of the device source (CPU) and on the H100: the output state against a float64 re-evaluation, the
    normal equations of Steps 1 and 2 against the float64 oracle, the Gauss-Newton solve at every n above the sizes the
    other modules reach, up to n2 + 8, and at the normal equations the linearisation exports;
  * on the H100: the drop-in float64 Stage II against the sequential float64 oracle, and Stage I with optimize_face (one
    linearisation against the oracle's rows at a given state, and a short run against the oracle).

Float32 bounds: 4x the maxima of the float32 host build over the same inputs, as ``TWIN_F32`` of
tests/test_gpu_normal_equations.py and ``TOL`` of tests/test_gpu_same_state.py were set.  The host build's maxima were
    normal equations (Step 1 / Step 2): J 3.6e-5 / 2.7e-4, r 3.0e-6, vp 7.2e-7, markers 3.0e-6 m, A 3.1e-5 / 8.2e-5, g 1.8e-5,
    SSE 1.5e-7 / 2.2e-7, data 5.2e-8;
    output state: markers 3.5e-6 m (the sum over 80 expression directions in float32; 6.8e-7 at 8), the rest within TOL.
"""
import copy
import ctypes as C

import numpy as np
import pytest

from conftest import EmuStageIBackend, dense_obs, gpu_solve, run_oracle
from moshpp_b200 import chmosh, lib, synth
from moshpp_b200 import stagei as product
from oracle import stagei as oracle
from test_gpu_gauss_newton import (THREADS, _bind, _maxima, expected_ok, layout_desc, solve_errors, spd_system,
                                   KAPPA)
from test_gpu_normal_equations import (PREC, _prepare, emu_lin, gpu_linearize, lin_inputs,  # noqa: F401 (emu_lin: a fixture)
                                       normal_equation_errors)
import test_gpu_normal_equations as ne
import test_gpu_same_state as ss
from test_gpu_same_state import same_state_errors
from test_stagei_face import _compare

FACE80 = 'CF80'
# float32 normal equations of the 80-expression family: 4x the host build's maxima (see the module docstring)
TWIN_F32_FACE80 = dict(J=2.7e-4, r=3.0e-6, vp=7.2e-7, markers=3.0e-6, A=8.2e-5, g=1.8e-5, sse=2.2e-7, data=5.2e-8)
SAME_STATE_F32_MARKERS = 4 * 3.5e-6


def face80_case(cases, **kw):
    return cases('CF', **synth.REFERENCE_FACE, **kw)


@pytest.fixture(autouse=True)
def _face80_bounds(monkeypatch):
    monkeypatch.setitem(ne.TWIN_F32, FACE80, TWIN_F32_FACE80)
    monkeypatch.setitem(ss.TOL, 'f32', dict(ss.TOL['f32'], markers=SAME_STATE_F32_MARKERS))


# ---- the fixture ------------------------------------------------------------------------------------------------------

def test_reference_face_fixture_has_the_reference_layout(cases):
    case = face80_case(cases)
    assert case['model']['shapedirs'].shape[-1] == 400
    sm = case['cfg'].surface_model
    assert (sm.betas_expr_start_id, sm.num_expressions) == (300, 80)
    pk, _, flags = chmosh.prepare_stageii(case['cfg'], case['markers_latent'], case['latent_labels'], case['betas'],
                                          case['marker_meta'])
    assert pk.n_expr == pk.n_dmpl == 80 and flags['n_betas_model'] == 400 and flags['expr_start'] == 300
    assert len(pk.free_step2) == len(cases('CF')['pack'].free_step2) + 72
    # the reference's expression output is the whole tail of the shape space from betas_expr_start_id
    res = lib.ResultArrays(2, lib.pack_dims(pk))
    res.status[:] = lib.ST_SOLVED
    obs, vis = dense_obs(case)
    data = chmosh.assemble_stageii_data(res, obs[:2], vis[:2], case['latent_labels'], pk, flags, False)
    assert data['expression'].shape == (2, 100)
    # the default fixture is unchanged: its own model file, 24 components, 8 expressions
    assert cases('CF')['model']['shapedirs'].shape[-1] == 24 and cases('CF')['pack'].n_expr == 8


# ---- the workspace plan -------------------------------------------------------------------------------------------------

# markers per type (body, fingers per hand, face) of the CF layout (65 markers) and of a denser one (90)
LAYOUTS = {65: dict(smpl=(65, 0, 0), smplh=(53, 6, 0), smplx=(41, 6, 12), mano=(0, 65, 0), animal_horse=(65, 0, 0)),
           90: dict(smpl=(90, 0, 0), smplh=(70, 10, 0), smplx=(56, 10, 14), mano=(0, 90, 0), animal_horse=(90, 0, 0))}
STAGEII = {'SMPL': ('C1', {}), 'SMPL-H': ('C2', {}), 'SMPL-X': ('C3', dict(optimize_dynamics=False)), 'SMPL-X+DMPL': ('C3', {}), 'SMPL-X-face80': ('CF', {}),
           'MANO': ('C4', {}), 'horse': ('CH', {})}
STAGEI = {'SMPL-H-betas16': 'C2', 'SMPL-X-betas16': 'C3', 'SMPL-X-face80': 'CF'}


def _relayout(case, n_markers):
    """The case's model and configuration with the marker layout of LAYOUTS[n_markers]."""
    mt = case['cfg'].surface_model.type
    nb, nf, nface = LAYOUTS[n_markers][mt]
    labels, vids, meta = synth.make_layout(case['model'], mt, nb, nf, n_face=nface)
    assert len(labels) == n_markers
    ml = synth.make_markers_latent(case['model'], mt, case['betas'], 16, vids, meta)
    return labels, meta, ml


def _stageii_pack(cases, config, flags, n_markers):
    case = face80_case(cases) if config == 'CF' else cases(config)
    cfg = copy.deepcopy(case['cfg'])
    cfg.moshpp.optimize_fingers = True
    for k, v in flags.items():
        cfg.moshpp[k] = v
    labels, meta, ml = _relayout(case, n_markers)
    pk, _, _ = chmosh.prepare_stageii(cfg, ml, labels, case['betas'], meta)
    return pk


class _NoBackend:
    pass


def _stagei_pack(cases, config, n_markers):
    case = face80_case(cases) if config == 'CF' else cases(config)
    cfg = copy.deepcopy(case['cfg'])
    cfg.moshpp.optimize_fingers = True
    cfg.moshpp.optimize_betas = config != 'CF'
    cfg.moshpp.optimize_face = config == 'CF'
    labels, meta, _ = _relayout(case, n_markers)
    frames = [{l: np.zeros(3) for l in labels}]
    s = product.StageI(frames, cfg, meta, betas=case['betas'] if config == 'CF' else None, backend=_NoBackend())
    pk = s.pack_for(True)
    assert pk.n_dmpl == (80 if config == 'CF' else 16) and pk.n_markers == n_markers
    return pk


@pytest.fixture(scope='module')
def emu_plan():
    from moshpp_b200 import build
    fn = C.CDLL(build.build_emu()).mosh2_emu_plan
    fn.argtypes = [C.POINTER(lib.ModelDesc), C.c_int32, C.c_int32, C.POINTER(C.c_int64)]
    fn.restype = C.c_int32

    def plan(pk, precision, multi):
        out = (C.c_int64 * 5)()
        assert fn(C.byref(lib.DescHolder(pk).desc), PREC[precision], multi, out) == 0
        return dict(smem=out[0], gws=out[1], big=out[2], tile=out[3], budget=out[4])
    return plan


def _assert_plans(emu_plan, pk, what):
    for precision in ('f32', 'f64'):
        for multi in (0, 1):
            p = emu_plan(pk, precision, multi)
            assert p['smem'] <= p['budget'], (what, precision, 'multi' if multi else 'single', p)


@pytest.mark.parametrize('n_markers', [65, 90])
@pytest.mark.parametrize('name', list(STAGEII))
def test_stageii_workspace_plan_fits(cases, emu_plan, name, n_markers):
    config, flags = STAGEII[name]
    pk = _stageii_pack(cases, config, flags, n_markers)
    _assert_plans(emu_plan, pk, (name, n_markers, len(pk.free_step2)))


@pytest.mark.parametrize('n_markers', [65, 90])
@pytest.mark.parametrize('name', list(STAGEI))
def test_stagei_workspace_plan_fits(cases, emu_plan, name, n_markers):
    pk = _stagei_pack(cases, STAGEI[name], n_markers)
    _assert_plans(emu_plan, pk, (name, n_markers, len(pk.free_step2)))


def test_face80_plan_is_the_global_workspace_layout(cases, emu_plan):
    """At 80 expressions both precisions need the global-workspace layout; the 8-expression CF float32 job keeps the shared
    one (the path the benchmark's SMPL-H family takes is covered by the SASS comparison, not here)."""
    pk = face80_case(cases)['pack']
    assert len(pk.free_step2) == 194
    for precision in ('f32', 'f64'):
        assert emu_plan(pk, precision, 0)['big'] == 1
    assert emu_plan(cases('CF')['pack'], 'f32', 0)['big'] == 0


# ---- output state and normal equations: host build (CPU) and kernel (H100) ----------------------------------------------

def _short(cases):
    return face80_case(cases, frames=10)


@pytest.mark.parametrize('precision', ['f64', 'f32'])
def test_device_source_face80_output_state_equals_float64_evaluation(cases, emu, precision):
    case = _short(cases)
    st = same_state_errors(case, emu(case, precision=PREC[precision]), precision)
    print(precision, {k: float('%.2g' % v) for k, v in st.items()})
    assert st['checked_velo'] > 0


@pytest.mark.parametrize('precision', ['f64', 'f32'])
@pytest.mark.parametrize('step', [1, 2])
def test_device_source_face80_normal_equations_equal_float64(cases, emu, emu_lin, step, precision):
    case = _short(cases)
    pk, opts = _prepare(case)
    obs, vis, x = lin_inputs(case, emu(case))
    out = emu_lin(pk, opts, obs, vis, x, step, precision)
    st = normal_equation_errors(case, FACE80, pk, opts, step, obs, vis, x, out, precision)
    print(step, precision, {k: float('%.2g' % v) for k, v in st.items()})


@pytest.mark.gpu
@pytest.mark.parametrize('precision', ['f64', 'f32'])
def test_kernel_face80_output_state_equals_float64_evaluation(cases, precision):
    case = _short(cases)
    st = same_state_errors(case, gpu_solve(case, precision=precision), precision)
    print(precision, {k: float('%.2g' % v) for k, v in st.items()})
    assert st['checked_velo'] > 0


@pytest.fixture(scope='module')
def face80_states():
    cache = {}

    def get(case):
        if 'x' not in cache:
            cache['x'] = lin_inputs(case, gpu_solve(case, precision='f64'))
        return cache['x']
    return get


@pytest.mark.gpu
@pytest.mark.parametrize('precision', ['f64', 'f32'])
@pytest.mark.parametrize('step', [1, 2])
def test_kernel_face80_normal_equations_equal_float64(cases, face80_states, step, precision):
    case = _short(cases)
    pk, opts = _prepare(case)
    obs, vis, x = face80_states(case)
    out = gpu_linearize(pk, opts, obs, vis, x, step, precision)
    # float32: the global-workspace layout, J^T J on the CUDA cores (no split-TF32 allowance)
    st = normal_equation_errors(case, FACE80, pk, opts, step, obs, vis, x, out, precision)
    print(step, precision, {k: float('%.2g' % v) for k, v in st.items()})


@pytest.mark.gpu
def test_f64_kernel_face80_equals_oracle(cases):
    """The drop-in call in float64 (the exact preset's precision) against the sequential float64 oracle, with the bounds of
    test_gpu_parity.test_f64_kernel_equals_oracle."""
    case = _short(cases)
    out = chmosh.mosh_stageii(mocap_fname=case['mocap_fname'], cfg=case['cfg'], markers_latent=case['markers_latent'],
                              latent_labels=case['latent_labels'], betas=case['betas'], marker_meta=case['marker_meta'],
                              precision='f64', chunk_len=0)
    ref = run_oracle(case)
    assert out['expression'].shape == ref['expression'].shape == (len(ref['fullpose']), 100)
    assert np.abs(out['expression'] - ref['expression']).max() < 1e-8
    assert np.abs(out['expression'][:, :80]).max() > 1e-3 and not np.any(out['expression'][:, 80:])
    assert np.abs(out['fullpose'] - ref['fullpose']).max() < 1e-8
    assert np.abs(out['trans'] - ref['trans']).max() < 1e-9
    dbg, rdbg = out['stageii_debug_details'], ref['stageii_debug_details']
    for k in ('data', 'poseB', 'poseF', 'expr'):
        assert np.allclose(dbg['stageii_errs'][k], rdbg['stageii_errs'][k], rtol=1e-7, atol=1e-10), k
    assert np.abs(np.concatenate(dbg['markers_sim']) - np.concatenate(rdbg['markers_sim'])).max() < 1e-9


# ---- Gauss-Newton at n above 136 and at the exported normal equations --------------------------------------------------

def _n2(cases):
    return len(face80_case(cases)['pack'].free_step2)


def check_sizes_above_136(run, cases, precision, big, threads):
    """Every n from 137 to n2 + 8 in the layout of a model with n free variables; the global-workspace layout must take
    every n."""
    st, refused = {}, []
    for n in range(137, _n2(cases) + 9):
        A, g = spd_system(n, precision, 3000 + n, KAPPA[precision] ** ((n % 4) / 3))
        assert expected_ok(A, precision) == 1
        rc, dgn, Ag, ok = run(precision, big, threads, layout_desc(n), A, g)
        if rc == -1:
            refused.append(n)
            continue
        assert ok == 1, n
        for k, v in solve_errors(A, g, dgn, Ag, precision).items():
            st[k] = max(st.get(k, 0.0), v)
    assert not big or not refused, refused
    assert refused == list(range(refused[0], _n2(cases) + 9)) if refused else True   # the layout grows with n
    return st


def check_face80_systems(run, lins, desc, precision):
    """The exported normal equations in the layout of the 80-expression model; it runs in the global-workspace layout."""
    st = {}
    for A, g in lins:
        exp = expected_ok(A, precision)
        assert exp is not None
        rc, dgn, Ag, ok = run(precision, 1, THREADS[precision], desc, A, g)
        assert rc == 0 and ok == exp
        if ok:
            for k, v in solve_errors(A, g, dgn, Ag, precision).items():
                st[k] = max(st.get(k, 0.0), v)
    return st


@pytest.fixture(scope='module')
def emu_gn():
    from moshpp_b200 import build
    return _bind(C.CDLL(build.build_emu()).mosh2_emu_gauss_newton)


@pytest.fixture(scope='module')
def gpu_gn():
    from moshpp_b200 import build
    return _bind(C.CDLL(build.build_gn_test()).gn_run)


@pytest.mark.parametrize('big', [0, 1])
@pytest.mark.parametrize('precision', ['f32', 'f64'])
def test_device_source_solves_sizes_above_136(cases, emu_gn, precision, big):
    print(precision, big, _maxima(check_sizes_above_136(emu_gn, cases, precision, big, THREADS[precision])))


@pytest.mark.parametrize('precision', ['f32', 'f64'])
@pytest.mark.parametrize('step', [1, 2])
def test_device_source_solves_the_face80_normal_equations(cases, emu, emu_lin, emu_gn, step, precision):
    case = _short(cases)
    pk, opts = _prepare(case)
    obs, vis, x = lin_inputs(case, emu(case))
    out = emu_lin(pk, opts, obs, vis, x, step, precision)
    st = check_face80_systems(emu_gn, zip(out['A'], out['g']), lib.DescHolder(pk).desc, precision)
    print(step, precision, _maxima(st))


GN_LAYOUTS = [(p, big, t) for p in ('f32', 'f64') for big in (0, 1) for t in ((128, 256, 384) if p == 'f32' else (128, 256))]


@pytest.mark.gpu
@pytest.mark.parametrize('precision,big,threads', GN_LAYOUTS)
def test_kernel_solves_sizes_above_136(cases, gpu_gn, precision, big, threads):
    print(precision, big, threads, _maxima(check_sizes_above_136(gpu_gn, cases, precision, big, threads)))


@pytest.mark.gpu
@pytest.mark.parametrize('precision', ['f32', 'f64'])
@pytest.mark.parametrize('step', [1, 2])
def test_kernel_solves_the_face80_normal_equations(cases, face80_states, gpu_gn, step, precision):
    case = _short(cases)
    pk, opts = _prepare(case)
    obs, vis, x = face80_states(case)
    out = gpu_linearize(pk, opts, obs, vis, x, step, precision)
    st = check_face80_systems(gpu_gn, zip(out['A'], out['g']), lib.DescHolder(pk).desc, precision)
    print(step, precision, _maxima(st))


# ---- Stage I with optimize_face at 80 expressions (the library linearises in float64) ------------------------------------

def face80_stagei_case(cases, tmp_path, n_pick=3):
    from conftest import stagei_case
    case, cfg, frames = stagei_case(cases, 'CF', n_pick, frames=40, dropout=0.02, **synth.REFERENCE_FACE)
    cfg.moshpp.optimize_betas = False
    fn = str(tmp_path / 'betas.npz')
    np.savez(fn, betas=case['betas'])
    return case, cfg, frames, fn


def _stagei_linearisation(backend, cases, tmp_path):
    """One Step-2 linearisation at a given state (non-zero jaw and expressions) against the oracle's J, r, A and g."""
    case, cfg, frames, _ = face80_stagei_case(cases, tmp_path)
    s = product.StageI(frames, cfg, case['marker_meta'], betas=case['betas'], backend=backend)
    assert s.face and s.ne == 80
    rng = np.random.default_rng(5)
    s.pose[:, :3] = rng.normal(0, 0.1, (s.F, 3))
    s.pose[:, 3:66] = rng.normal(0, 0.05, (s.F, 63))
    s.pose[:, 66:69] = rng.normal(0, 0.2, (s.F, 3))
    s.trans[:] = rng.normal(0, 0.01, (s.F, 3)) + np.array([0.0, 0.9, 0.0])
    s.expr[:] = rng.normal(0, 0.5, s.expr.shape)
    wts = s.weights_for(0.25)
    pk = s.pack_for(True, s.can(s.betas[:s.nb]))
    x = np.zeros((s.F, pk.nx))
    x[:, :3], x[:, 3:3 + pk.p_red], x[:, 3 + pk.p_red:] = s.trans, s.pose, s.expr
    opts = lib.make_options(None, optimize_fingers=True, optimize_face=True)
    opts.wt_data, opts.wt_poseB, opts.wt_poseH = wts['data'], wts['poseB'], wts['poseH']
    opts.wt_poseF, opts.wt_expr = wts['poseF'], wts['expr']
    dev = backend.linearize(pk, opts, s.obs, s.vis, x, 2, True)

    o = oracle.StageISolver(frames, cfg, case['marker_meta'], case['betas'])
    ids = o.pose_ids_for(True)
    o.pose[:], o.trans[:], o.expr[:] = s.pose, s.trans, s.expr
    _, off_ml, off_fr, per, n = o.layout(ids, False, True)
    assert per == len(pk.free_step2)
    free = [0, 1, 2] + [3 + int(i) for i in ids]
    assert list(pk.free_step2[:len(free)]) == free
    M, F = o.n_markers, s.F
    col = {l: i for i, l in enumerate(s.labels)}
    at = {}
    r_all, J_all = o.residual(o.get_x(ids, False, True), True, ids, False, o.weights_for(0.25), True, free_expr=True,
                              rows=at)
    # the oracle's rows of every frame: its data rows, its poseF rows (3 per frame) and its expr rows (80 per frame)
    nv = [len(i) for i in o.lm_ids]
    data0, poseF0, expr0 = at['data'].start, at['poseF'].start, at['expr'].start
    sel = np.r_[np.arange(3), 3 + len(ids) + np.arange(80)]          # translation and expressions: data and expr terms only
    for f in range(F):
        rows = np.arange(data0 + 3 * sum(nv[:f]), data0 + 3 * sum(nv[:f + 1]))
        cols = slice(off_fr + f * per, off_fr + (f + 1) * per)
        slots = (3 * np.asarray([col[l] for l in np.asarray(o.latent_labels)[o.lm_ids[f]]])[:, None] + np.arange(3)).ravel()
        Jref, rref = np.zeros((3 * M, per)), np.zeros(3 * M)
        Jref[slots] = -J_all[rows][:, cols]            # the oracle's r = obs - sim, the kernel's r = sim - obs
        rref[slots] = -r_all[rows]
        assert np.abs(dev['J'][f] - Jref).max() <= 1e-9 * np.abs(Jref).max(), f
        assert np.abs(dev['r'][f] - rref).max() <= 1e-9 * np.abs(rref).max(), f
        own = np.r_[rows, poseF0 + 3 * f + np.arange(3), expr0 + 80 * f + np.arange(80)]
        Jf, rf = J_all[own][:, cols], r_all[own]
        A_ref, g_ref = Jf.T @ Jf, -Jf.T @ rf
        d = np.sqrt(np.diag(A_ref))[sel]
        assert np.abs((dev['A'][f] - A_ref)[np.ix_(sel, sel)] / np.outer(d, d)).max() <= 1e-9, f
        assert np.abs(dev['g'][f][sel] - g_ref[sel]).max() <= 1e-9 * np.abs(g_ref[sel]).max(), f
    return dev


def test_device_source_face80_stagei_linearisation_equals_oracle(cases, tmp_path):
    _stagei_linearisation(EmuStageIBackend(), cases, tmp_path)


@pytest.mark.gpu
def test_kernel_face80_stagei_linearisation_equals_oracle(cases, tmp_path):
    _stagei_linearisation(product.DeviceBackend(), cases, tmp_path)


@pytest.mark.gpu
def test_face80_stagei_on_the_gpu_equals_oracle(cases, tmp_path):
    case, cfg, frames, fn = face80_stagei_case(cases, tmp_path)
    cfg.opt_settings.maxiter = 4
    ref = oracle.mosh_stagei(frames, cfg, betas_fname=fn, marker_meta=case['marker_meta'])
    out = product.mosh_stagei(frames, cfg, betas_fname=fn, marker_meta=case['marker_meta'])
    _compare(out, ref, 1e-6)
    assert np.stack(out['stagei_debug_details']['opt_models_expression']).shape == (len(frames), 80)
