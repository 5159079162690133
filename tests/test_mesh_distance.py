"""Stage-I surface term (SURVEY.md 8(f-2)): point-to-triangle-mesh distance with derivatives.

CPU: the oracle's restatement against the reference header itself (vectors of the UNMODIFIED
scan2mesh/mesh_distance/sample2meshdist.h, compiled against an Eigen stand-in by oracle/build_ref.py, stored in
tests/golden/ref_s2m.npz by make_reference_vectors.py) and against finite differences.  GPU: the CUDA kernel (C-ABI
mosh2_mesh_distance) against the oracle."""
import os

import numpy as np
import pytest

from oracle import mesh_distance as omd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _random_case(rng):
    a, b, c = rng.normal(0, 0.3, (3, 3))
    x = (a + b + c) / 3 + rng.normal(0, 0.2, 3)
    return x, a, b, c


def test_oracle_tri_equals_reference_header():
    """Every part (plane, three edges, three vertices) under the three robustifiers: value and all four gradients."""
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'ref_s2m.npz'))
    assert [(int(k), s) for k, s in g['kinds']] == [(omd.KIND_DISTANCE, 1.0), (omd.KIND_SQUARED, 1.0), (omd.KIND_GM, 0.05), (omd.KIND_GM, 0.5)]
    rng = np.random.default_rng(7)
    for trial in range(40):
        x, a, b, c = _random_case(rng)
        assert np.array_equal(np.stack([x, a, b, c]), g['xabc'][trial])          # same inputs as the reference saw
        for ki, (kind, sigma) in enumerate(g['kinds']):
            for part in range(7):
                rv, rgrad = g['value'][trial, ki, part], g['grad'][trial, ki, part]
                got = omd.tri(part, x, a, b, c, int(kind), float(sigma))
                assert abs(got[0] - rv) <= 1e-12 * max(1.0, abs(rv))
                for gg, r in zip(got[1:], rgrad):
                    assert np.abs(gg - r).max() <= 1e-10 * max(1.0, np.abs(r).max()), (kind, part)


def test_oracle_gradients_are_derivatives():
    rng = np.random.default_rng(11)
    for trial in range(10):
        x, a, b, c = _random_case(rng)
        for kind, sigma in ((omd.KIND_SQUARED, 1.0), (omd.KIND_GM, 0.1)):
            for part in range(7):
                v, dx, da, db, dc = omd.tri(part, x, a, b, c, kind, sigma)
                for which, g in enumerate((dx, da, db, dc)):
                    num = np.zeros(3)
                    for k in range(3):
                        args = [x.copy(), a.copy(), b.copy(), c.copy()]
                        args[which][k] += 1e-6
                        vp = omd.tri(part, *args, kind, sigma)[0]
                        args[which][k] -= 2e-6
                        vm = omd.tri(part, *args, kind, sigma)[0]
                        num[k] = (vp - vm) / 2e-6
                    assert np.abs(num - g).max() < 1e-6 * max(1.0, np.abs(g).max())


def test_nearest_part_is_consistent_with_the_distance():
    """The brute-force query returns the triangle / part whose closed-form distance (of that part) is the minimum over all
    triangles -- what the AABB tree of the reference returns (mesh_distance_main.py:358-376)."""
    rng = np.random.default_rng(3)
    verts = rng.normal(0, 0.3, (60, 3))
    faces = rng.integers(0, 60, (150, 3))
    faces = faces[(faces[:, 0] != faces[:, 1]) & (faces[:, 1] != faces[:, 2]) & (faces[:, 0] != faces[:, 2])]
    # an isolated triangle far from the soup, with samples beyond its corners and edges: vertex and edge parts for sure
    verts = np.concatenate([verts, [[10, 0, 0], [11, 0, 0], [10, 1, 0]]])
    faces = np.concatenate([faces, [[60, 61, 62]]])
    corner = np.array([[9.5, -0.5, 0.2], [11.8, -0.3, 0.1], [9.7, 1.9, -0.2], [10.5, -0.7, 0.1], [11.0, 1.0, 0.3], [9.2, 0.5, 0.0]])
    samples = np.concatenate([rng.normal(0, 0.35, (50, 3)), corner])
    r, dsample, dref, t, p = omd.somedistance(samples, verts, faces, omd.KIND_DISTANCE)
    assert p[-6:].tolist() == [4, 5, 6, 1, 2, 3] and (t[-6:] == len(faces) - 1).all()
    parts = set(np.unique(p).tolist())
    assert 0 in parts and parts & {1, 2, 3} and parts & {4, 5, 6}      # interior, edge and vertex cases all occur
    for s in range(len(samples)):
        a, b, c = (verts[faces[t[s], k]] for k in range(3))
        assert abs(abs(r[s]) - abs(omd.tri(int(p[s]), samples[s], a, b, c)[0])) < 1e-12
        A, B, Cc = verts[faces[:, 0]], verts[faces[:, 1]], verts[faces[:, 2]]
        d2, _ = omd.closest_on_triangles(samples[s], A, B, Cc)
        assert abs(np.sqrt(d2.min()) - abs(r[s])) < 1e-9
        assert np.abs(dsample[s] + dref[s].reshape(3, 3).sum(0)).max() < 1e-9      # translation invariance


# Shapes of the GPU search (S samples, about T triangles) and the path of nearest_kernel each is there for, on an H100's
# 132 SMs: blocks of 128 samples x triangle ranges of whole 384-triangle tiles, four blocks per SM (mosh2.cu).
SHAPES = {
    (1, 1): 'one partial sample block, one tile of one triangle',
    (129, 385): 'two sample blocks, the second partial; two ranges, the second a partial tile of one triangle',
    (333, 1300): 'the former single shape plus a duplicated triangle, a collinear one and all seven parts',
    (4096, 20000): '53 tiles in 14 ranges of 4 tiles: both ring stages refill and the mbarrier parity flips; last range 32',
}
EDGE_CASE = (333, 1300)
N_PLACED = 13          # hand-placed samples at the end of the edge case

def _split(S, T, n_sm, spb=128, tile=384):
    """The host's grid of nearest_kernel (mosh2_mesh_distance): (sample blocks, ranges, triangles per range)."""
    sblocks = (S + spb - 1) // spb
    splits = (4 * max(n_sm, 1) + sblocks - 1) // sblocks
    tiles = (T + tile - 1) // tile
    splits = max(1, min(splits, tiles))
    per = ((tiles + splits - 1) // splits) * tile
    return sblocks, (T + per - 1) // per, per


def _mesh_case(S, T):
    rng = np.random.default_rng(5)
    if T == 1:
        return np.array([[0.0, 0, 0], [1, 0.1, 0], [0.2, 0.9, 0.1]]), np.array([[0, 1, 2]], dtype=np.int32), np.array([[0.3, 0.3, 0.2]])
    V = max(3, T // 2)
    verts = rng.normal(0, 0.3, (V, 3))
    faces = rng.integers(0, V, (int(T * 1.1), 3)).astype(np.int32)
    faces = faces[(faces[:, 0] != faces[:, 1]) & (faces[:, 1] != faces[:, 2]) & (faces[:, 0] != faces[:, 2])][:T]
    samples = [rng.normal(0, 0.35, (S, 3))]
    if (S, T) == EDGE_CASE:
        # an isolated triangle (and a duplicate of it) away from the soup, and a collinear triangle: zero area, no zero edge
        a, b, c = np.array([2.0, 0.1, 0.0]), np.array([3.0, 0.0, 0.05]), np.array([2.2, 0.9, 0.0])
        p, q, m = np.array([2.0, 2.0, 0.0]), np.array([3.0, 2.4, 0.2]), np.array([2.25, 2.1, 0.05])
        n0 = len(verts)
        verts = np.concatenate([verts, [a, b, c, p, q, m]])
        faces = np.concatenate([faces, [[n0, n0 + 1, n0 + 2], [n0, n0 + 1, n0 + 2], [n0 + 3, n0 + 4, n0 + 5]]]).astype(np.int32)
        nrm = np.cross(b - a, c - a)
        nrm /= np.linalg.norm(nrm)
        cen = (a + b + c) / 3
        near = [cen + 1e-3 * nrm]                                                  # plane
        for u, v in ((a, b), (b, c), (c, a)):                                      # 1e-3 beyond each edge, in the plane
            out = np.cross(v - u, nrm)
            out /= np.linalg.norm(out)
            if np.dot(out, cen - u) > 0:
                out = -out
            near.append((u + v) / 2 + 1e-3 * out)
        for u in (a, b, c):                                                        # 1e-3 beyond each vertex
            near.append(u + 1e-3 * (u - cen) / np.linalg.norm(u - cen))
        line = (q - p) / np.linalg.norm(q - p)                                     # around the collinear triangle
        side = np.cross(line, [0.0, 0.0, 1.0])
        for s in (0.1, 0.3, 0.6, 0.9):
            near.append(p + s * (q - p) + 1e-3 * side + 2e-4 * np.array([0, 0, 1.0]))
        near += [p - 1e-3 * line, q + 1e-3 * line]
        samples = [samples[0][:S - len(near)], np.array(near)]
    return verts, faces, np.concatenate(samples)


_BRUTE = {}


def _brute(key):
    """float64 brute force over all triangles: the nearest (triangle, part), the squared distance, and the float32
    rounding scale of every (sample, triangle) pair of closest_part (see test_cuda_mesh_distance_equals_oracle)."""
    if key not in _BRUTE:
        verts, faces, samples = _mesh_case(*key)
        A, B, C = verts[faces[:, 0]], verts[faces[:, 1]], verts[faces[:, 2]]
        scale = np.linalg.norm(B - A, axis=1) + np.linalg.norm(C - A, axis=1) + np.linalg.norm(A, axis=1)   # (L without p)
        d2min = np.zeros(len(samples))
        t = np.zeros(len(samples), dtype=np.int64)
        p = np.zeros(len(samples), dtype=np.int64)
        for s, x in enumerate(samples):           # (omd.nearest, keeping the distance)
            d2, part = omd.closest_on_triangles(x, A, B, C)
            t[s] = np.argmin(d2)
            d2min[s], p[s] = d2[t[s]], part[t[s]]
        _BRUTE[key] = dict(verts=verts, faces=faces, samples=samples, d2min=d2min, tri=t, part=p, scale=scale)
    return _BRUTE[key]


def test_mesh_distance_shapes_reach_their_paths():
    """The brute force of the GPU test's smaller shapes: every float64 distance finite, all seven parts in the edge case;
    and on 132 SMs the grid each shape is there for."""
    for key in list(SHAPES)[:3]:
        b = _brute(key)
        assert len(b['samples']) == key[0] and abs(len(b['faces']) - key[1]) <= 3
        assert np.isfinite(b['d2min']).all()
    assert set(_brute(EDGE_CASE)['part'].tolist()) == set(range(7))
    assert _split(1, 1, 132) == (1, 1, 384)
    assert _split(129, 385, 132) == (2, 2, 384)
    sb, splits, per = _split(4096, 20000, 132)
    assert (sb, splits, per, 20000 - (splits - 1) * per) == (32, 14, 1536, 32)


@pytest.mark.gpu
@pytest.mark.parametrize('kind,sigma', [(omd.KIND_DISTANCE, 1.0), (omd.KIND_SQUARED, 1.0), (omd.KIND_GM, 0.05)])
def test_cuda_mesh_distance_equals_oracle(kind, sigma):
    """Every sample, every shape of SHAPES.  The search runs in float32 and may return another (triangle, part) than the
    float64 brute force where two are within round-off; so for EVERY sample the float64 distance of the part the GPU
    returned, d_gpu, must equal the brute-force minimum d* over all triangles within the float32 rounding of
    closest_part.  That computes q = p - (closest point of the region) from float32 inputs (sample and vertices each
    rounded by 2^-24 |.|) through differences and convex combinations of vectors no longer than
    L = |p| + |a| + |p - a| + |b - a| + |c - a|, so |q_float32 - q| <= c 2^-24 L, and | |q_float32| - |q| | is no larger.
    The GPU keeps the smallest |q_float32|; hence |d_gpu - d*| <= c 2^-24 (L_gpu + L_ref), c = 16, with L of the GPU's
    and of the brute force's triangle.  The check is two-sided: a plane distance taken where the closest point is on an
    edge is too small, another triangle's distance too large.  Where the GPU and the brute force agree on (triangle,
    part), value and derivatives equal the oracle's to 1e-12 / 1e-9."""
    import torch
    from moshpp_b200 import mesh_distance as md
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    for key in SHAPES:
        b = _brute(key)
        verts, faces, samples = b['verts'], b['faces'], b['samples']
        if n_sm == 132 and key == (4096, 20000):
            sb, splits, per = _split(len(samples), len(faces), n_sm)
            assert (splits, per // 384) == (14, 4)
        out = md.mesh_distance(samples, verts, faces, kind=kind, sigma=sigma)
        for k in ('value', 'd_sample', 'd_tri'):
            assert np.isfinite(out[k]).all(), (key, k)
        t, p = b['tri'], b['part']
        r, dsample, dref, _, _ = omd.somedistance(samples, verts, faces, kind, sigma, nearest_tri=t, nearest_part=p)
        # every sample: the float64 distance of the GPU's (triangle, part) against the brute-force minimum
        L = lambda tt, x: b['scale'][tt] + np.linalg.norm(x) + np.linalg.norm(x - verts[faces[tt, 0]])
        for s in range(len(samples)):
            tg, pg = int(out['tri'][s]), int(out['part'][s])
            a, bb, c = (verts[faces[tg, q]] for q in range(3))
            with np.errstate(all='ignore'):
                d_gpu = abs(omd.tri(pg, samples[s], a, bb, c, omd.KIND_DISTANCE)[0])
            bound = 16 * 2.0 ** -24 * (L(tg, samples[s]) + L(t[s], samples[s]))
            d_ref = np.sqrt(b['d2min'][s])
            assert abs(d_gpu - d_ref) <= bound, (key, s, tg, pg, t[s], p[s], d_gpu, d_ref, bound)
        same = (out['tri'] == t) & (out['part'] == p)
        if key == EDGE_CASE:
            # the samples around the isolated triangle are unambiguous (its duplicate ties: the lower index wins);
            # around the collinear one, edges on the same line tie
            assert same[-N_PLACED:-N_PLACED + 7].all()
        sc = max(1.0, np.abs(r).max())
        assert np.abs(np.abs(out['value']) - np.abs(r)).max() < 1e-5 * sc
        assert np.abs(out['value'][same] - r[same]).max() < 1e-12 * sc
        assert np.abs(out['d_sample'][same] - dsample[same]).max() < 1e-9 * max(1.0, np.abs(dsample).max())
        assert np.abs(out['d_tri'][same] - dref[same]).max() < 1e-9 * max(1.0, np.abs(dref).max())
        # with the nearest (triangle, part) given -- what the reference's somedistance takes -- everything is exact
        out2 = md.mesh_distance(samples, verts, faces, kind=kind, sigma=sigma, nearest_tri=t, nearest_part=p)
        assert np.abs(out2['value'] - r).max() < 1e-12 * sc
        assert np.abs(out2['d_tri'] - dref).max() < 1e-9 * max(1.0, np.abs(dref).max())
        V = len(verts)
        Dr_ref, Dr_sample = md.as_sparse(out2, faces, V)
        assert Dr_ref.shape == (len(samples), 3 * V) and Dr_sample.shape == (len(samples), 3 * len(samples))
        assert np.allclose(np.asarray(Dr_sample.sum(1)).ravel(), dsample.sum(1), atol=1e-9)
