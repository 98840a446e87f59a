"""CPU emulation of the shared core (embree_b200/csrc/rt_core.cuh compiled for the host by tests/emu): the LBVH
node construction, BVH8 collapse / slot assignment / 8-bit box quantisation, the traversal loop and the triangle
test are the exact routines the CUDA kernels call per thread.  They are checked against the oracle on small scenes
so logic errors surface without a GPU."""
import ctypes as C

import numpy as np
import pytest

from embree_b200 import scenes
from embree_b200.rtc import make_rayhits, rays_of
from tests.conftest import GOLDEN, load_golden
from tests.curve_cases import CURVE_KINDS
from tests.parity import compare_hits


def _emu_trace(emu, v, t, rays, occluded=False, mask=0xFFFFFFFF, policy=3, robust=False):
    v = np.ascontiguousarray(v, np.float32)
    t = np.ascontiguousarray(t, np.uint32)
    h = emu.emu_build(v.ctypes.data, len(v), t.ctypes.data, len(t), 0, mask, policy | (0x100 if robust else 0))
    stats = np.zeros(2, np.uint64)
    emu.emu_trace(h, rays.ctypes.data, len(rays), 1 if occluded else 0, stats.ctypes.data)
    info = dict(nodes=emu.emu_num_nodes(h), depth=emu.emu_depth(h), trav_nodes=int(stats[0]), trav_tris=int(stats[1]))
    emu.emu_free(h)
    return rays, info


@pytest.mark.parametrize("num_phi", [3, 8, 33])
def test_sphere_matches_oracle(emu, oracle, num_phi):
    v, t = scenes.triangle_sphere(num_phi)
    rays = scenes.as_numpy_rayhits(scenes.incoherent_rays_reference(5000))
    want = oracle.trace(v, t, rays.copy())
    got, info = _emu_trace(emu, v, t, rays.copy())
    rep = compare_hits(want, got)
    assert rep["id_mismatch"] == 0 and rep["tie"] == 0 and rep["hit_miss_disagree"] == 0, (rep, info)
    assert rep["max_rel_t"] == 0.0 and rep["ng_bit_exact"], rep  # same arithmetic -> same bits
    wo = oracle.trace(v, t, rays_of(rays), occluded=True)
    go, _ = _emu_trace(emu, v, t, rays_of(rays), occluded=True)
    assert (wo["tfar"].view(np.uint32) == go["tfar"].view(np.uint32)).all()


@pytest.mark.parametrize("robust", [False, True])
@pytest.mark.parametrize("policy", [0, 3])
def test_golden_single_mesh(emu, policy, robust):
    """Both collapse policies (greedy / SAH-optimal DP) and both intersectors (Moeller-Trumbore / robust Pluecker)."""
    meshes, rin, want_i, want_o, _ = load_golden("sphere21", robust)
    (v, t, gid, mask) = meshes[0]
    got, _ = _emu_trace(emu, v, t, rin.copy(), mask=mask, policy=policy, robust=robust)
    rep = compare_hits(want_i, got)
    assert rep["id_mismatch"] == 0 and rep["hit_miss_disagree"] == 0 and rep["max_rel_t"] <= 1e-4 and rep["ng_bit_exact"], rep
    go, _ = _emu_trace(emu, v, t, rays_of(rin), occluded=True, mask=mask, policy=policy, robust=robust)
    assert (go["tfar"].view(np.uint32) == want_o["tfar"].view(np.uint32)).all()


def test_robust_is_watertight(emu):
    """RTC_SCENE_FLAG_ROBUST: the Pluecker edge tests are watertight -- no ray from inside a closed mesh escapes."""
    v, t = scenes.triangle_sphere(50)
    rays = scenes.as_numpy_rayhits(scenes.incoherent_rays_reference(100000, org=(0.1, -0.2, 0.05)))
    got, _ = _emu_trace(emu, v, t, rays, robust=True)
    assert (got["geomID"] == 0).all()


def test_tiny_scenes(emu, oracle):
    """1, 2, 3, 4, 9 triangles: root-only trees, partially filled nodes."""
    rng = np.random.RandomState(5)
    for n in (1, 2, 3, 4, 9, 25):
        v = rng.uniform(-1, 1, (3 * n, 3)).astype(np.float32)
        t = np.arange(3 * n, dtype=np.uint32).reshape(n, 3)
        org = rng.uniform(-2, 2, (2000, 3)).astype(np.float32)
        d = (rng.uniform(-1, 1, (2000, 3)) - org * 0.5).astype(np.float32)
        rays = make_rayhits(org, d)
        want = oracle.trace(v, t, rays.copy())
        got, info = _emu_trace(emu, v, t, rays.copy())
        rep = compare_hits(want, got)
        assert rep["id_mismatch"] == 0 and rep["hit_miss_disagree"] == 0 and rep["tie"] == 0, (n, rep)


def test_axis_aligned_and_degenerate(emu, oracle):
    """Flat boxes (axis-aligned cube faces), zero direction components, degenerate (zero-area) triangles."""
    (cv, ct), _ = scenes.cube_and_ground()
    extra_v = np.array([[0, 0, 0], [0, 0, 0], [0, 0, 0], [3, 3, 3], [3, 3, 3], [4, 4, 4]], np.float32)
    v = np.concatenate([cv, extra_v])
    t = np.concatenate([ct, np.array([[8, 9, 10], [11, 12, 13]], np.uint32)])
    org = np.array([[0.3, 0.2, -5], [0.3, 0.2, 5], [-5, 0.1, 0.2], [0.5, 5, 0.5], [1, 1, -5], [0, 0, 0], [0.25, -5, 0.25]], np.float32)
    d = np.array([[0, 0, 1], [0, 0, -1], [1, 0, 0], [0, -1, 0], [0, 0, 1], [1, 1, 1], [0, 1, 0]], np.float32)
    rays = make_rayhits(org, d)
    want = oracle.trace(v, t, rays.copy())
    got, _ = _emu_trace(emu, v, t, rays.copy())
    rep = compare_hits(want, got)
    assert rep["id_mismatch"] == 0 and rep["hit_miss_disagree"] == 0, rep
    assert (want["geomID"][:4] == 0).all()


def test_watertight_sphere_from_inside(emu):
    """WatertightTest (verify.cpp:3611-3690): rays from inside a closed sphere must not leak (<= 2e-5)."""
    v, t = scenes.triangle_sphere(50)
    rays = scenes.as_numpy_rayhits(scenes.incoherent_rays_reference(50000, org=(0.1, -0.2, 0.05)))
    got, _ = _emu_trace(emu, v, t, rays)
    assert (got["geomID"] == 0xFFFFFFFF).mean() <= 2e-5


def test_nan_inf_rays_terminate(emu):
    """NaNTest/InfTest (verify.cpp:3813-3963): invalid rays must terminate and leave a miss."""
    v, t = scenes.triangle_sphere(8)
    bad = [np.nan, np.inf, -np.inf]
    org, d = [], []
    for b in bad:
        org += [[b, 0, 0], [0, 0, 0], [0, b, 0]]
        d += [[0, 0, 1], [b, 0, 1], [1, b, b]]
    rays = make_rayhits(np.array(org, np.float32), np.array(d, np.float32))
    _emu_trace(emu, v, t, rays)  # must return


def test_op_log_matches_traversal_counters(emu):
    """The operation log used by the offline warp-scheduling model (scripts/warp_model.py) has one 'N' per node step and
    one 'T' per triangle test of the production traversal, and the exact front-to-back variant finds the same hits."""
    import ctypes as C
    emu.emu_trace_ops.restype = C.c_uint64
    emu.emu_trace_ops.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64]
    emu.emu_trace_sorted.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
    v, t = scenes.triangle_sphere(64)
    h = emu.emu_build(v.ctypes.data, len(v), t.ctypes.data, len(t), 0, 0xFFFFFFFF, 3)
    rng = np.random.RandomState(2)
    org = (rng.normal(size=(20000, 3)) * 0.3).astype(np.float32)
    rays = make_rayhits(org, rng.normal(size=(20000, 3)).astype(np.float32))
    base, st = rays.copy(), np.zeros(2, np.uint64)
    emu.emu_trace(h, base.ctypes.data, len(base), 0, st.ctypes.data)
    ops = np.zeros(len(rays) * 256, np.uint8)
    n = emu.emu_trace_ops(h, rays.copy().ctypes.data, len(rays), ops.ctypes.data, len(ops))
    ops = ops[:n]
    assert (ops == 0).sum() == len(rays) and (ops == ord("N")).sum() == st[0] and (ops == ord("T")).sum() == st[1]
    got, s2 = rays.copy(), np.zeros(2, np.uint64)
    emu.emu_trace_sorted(h, got.ctypes.data, len(got), s2.ctypes.data)
    assert (base["primID"] == got["primID"]).mean() > 0.9999 and s2[0] <= st[0]
    emu.emu_free(h)


def test_curve_segment_test_equals_oracle(emu, oracle):
    """rt_core.cuh curve_test (the routine the device runs per round-linear-curve record, here compiled for the host) finds,
    by brute force over all segments, bit-identical t / u / Ng to the C oracle's BVH traversal on the golden curve rays --
    every operation is explicitly rounded, so device, host instantiation and oracle evaluate the same expressions."""
    import ctypes as C
    from tests.conftest import load_golden_curves
    g = load_golden_curves()
    cv, ci, cf, gid, mask = g["curves"][0][:5]
    sc = oracle.scene([], curves=[(cv, ci, cf, gid, 0xFFFFFFFF)])
    rays = g["rays_in"][::6].copy()
    rays["mask"] = 0xFFFFFFFF
    want = sc.trace(rays.copy())
    n = len(ci)
    right = np.zeros(n, bool)
    right[:-1] = ci[1:] == ci[:-1] + 1
    left = np.zeros(n, bool)
    left[1:] = right[:-1]
    P = lambda a: np.ascontiguousarray(a, np.float32).ctypes.data_as(C.c_void_p)   # noqa: E731
    out = (C.c_float * 5)()
    hits = 0
    for k in range(len(rays)):
        r = rays[k]
        ray = np.array([r["org_x"], r["org_y"], r["org_z"], r["tnear"], r["dir_x"], r["dir_y"], r["dir_z"], r["tfar"]], np.float32)
        best = None
        for i in range(n):
            v = int(ci[i])
            vL, vR = (cv[v - 1] if left[i] else cv[v]), (cv[v + 2] if right[i] else cv[v + 1])
            if emu.emu_curve_test(P(ray), P(cv[v]), P(cv[v + 1]), int(left[i]), P(vL), int(right[i]), P(vR), out):
                best = (out[0], out[1], out[2], out[3], out[4], i)
                ray[7] = out[0]                     # an accepted hit shrinks tfar for the following segments
        w = want[k]
        if best is None:
            assert w["geomID"] == 0xFFFFFFFF, k
            continue
        hits += 1
        got = np.array(best[:5], np.float32).view(np.uint32)
        exp = np.array([w["tfar"], w["u"], w["Ng_x"], w["Ng_y"], w["Ng_z"]], np.float32).view(np.uint32)
        assert (got == exp).all(), (k, best, w)
    assert hits > 100
    sc.free()


def test_flat_curve_segment_test_equals_oracle(emu, oracle):
    """rt_core.cuh flat_curve_test (RTC_GEOMETRY_TYPE_FLAT_LINEAR_CURVE), host instantiation, by brute force over all segments:
    bit-identical t / u / Ng to the C oracle on the golden rays."""
    import ctypes as C
    from tests.conftest import load_golden_curves
    g = load_golden_curves("curves_flat")
    cv, ci, cf, gid, mask, flat = g["curves"][0]
    sc = oracle.scene([], curves=[(cv, ci, cf, gid, 0xFFFFFFFF, True)])
    rays = g["rays_in"][::5].copy()
    rays["mask"] = 0xFFFFFFFF
    want = sc.trace(rays.copy())
    P = lambda a: np.ascontiguousarray(a, np.float32).ctypes.data_as(C.c_void_p)   # noqa: E731
    out = (C.c_float * 5)()
    hits = 0
    for k in range(len(rays)):
        r = rays[k]
        ray = np.array([r["org_x"], r["org_y"], r["org_z"], r["tnear"], r["dir_x"], r["dir_y"], r["dir_z"], r["tfar"]], np.float32)
        best = None
        for i in range(len(ci)):
            v = int(ci[i])
            if emu.emu_flat_curve_test(P(ray), P(cv[v]), P(cv[v + 1]), out):
                best = (out[0], out[1], out[2], out[3], out[4])
                ray[7] = out[0]
        w = want[k]
        if best is None:
            assert w["geomID"] == 0xFFFFFFFF, k
            continue
        hits += 1
        got = np.array(best, np.float32).view(np.uint32)
        exp = np.array([w["tfar"], w["u"], w["Ng_x"], w["Ng_y"], w["Ng_z"]], np.float32).view(np.uint32)
        assert got[0] == exp[0], (k, best, w)          # same distance; on an exact tie at a joint u / Ng name the other segment
        if not (got == exp).all():
            assert best[1] in (0.0, 1.0) and w["u"] in (0.0, 1.0), (k, best, w)
    assert hits > 100
    sc.free()


@pytest.mark.parametrize("which", [0, 1, 2, 3])
def test_flat_cubic_curve_test_equals_oracle(emu, oracle, which):
    """rt_core.cuh flat_cubic_test + curve_basis_table (flat Bezier / B-spline / Catmull-Rom / Hermite curves), host instantiation,
    brute force over all curves of one golden curve set: the same winner and bit-identical t / u / v / Ng as the C oracle's
    BVH traversal (an exact tie between two curves may name either)."""
    import ctypes as C
    from tests.conftest import load_golden_cubic
    from tests.parity import CUBIC_BASES
    g = load_golden_cubic()
    cv, ci, gid, mask, basis, tess, tang = g["cubics"][which][:7]
    tess = 4 if tess is None else tess
    sc = oracle.scene([], cubics=[(cv, ci, gid, 0xFFFFFFFF, basis, tess, tang)])
    rays = g["rays_in"][::2].copy()
    rays["mask"] = 0xFFFFFFFF
    want = sc.trace(rays.copy())
    if basis == "hermite":    # the conversion HermiteCurveT does (hermite_curve.h:19-20), with the same fused operations
        k = np.float32(1.0 / 3.0)
        fma = lambda a, b, c: (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)   # noqa: E731
        p0, p1, t0, t1 = cv[ci], cv[ci + 1], tang[ci], tang[ci + 1]
        cps = np.stack([p0, fma(np.full_like(t0, k), t0, p0), fma(np.full_like(t1, -k), t1, p1), p1], 1)
    else:
        cps = np.stack([cv[ci + j] for j in range(4)], 1)
    cps = np.ascontiguousarray(cps, np.float32)
    emu.emu_flat_cubic_closest.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_uint, C.c_int, C.c_void_p]
    out = (C.c_float * 6)()
    hits = 0
    for k in range(len(rays)):
        r = rays[k]
        ray = np.array([r["org_x"], r["org_y"], r["org_z"], r["tnear"], r["dir_x"], r["dir_y"], r["dir_z"], r["tfar"]], np.float32)
        win = emu.emu_flat_cubic_closest(ray.ctypes.data, cps.ctypes.data, len(ci), 0 if basis == "hermite" else CUBIC_BASES.index(basis), tess, out)
        w = want[k]
        if win < 0:
            assert w["geomID"] == 0xFFFFFFFF, k
            continue
        hits += 1
        got = np.array(list(out), np.float32).view(np.uint32)
        exp = np.array([w["tfar"], w["u"], w["v"], w["Ng_x"], w["Ng_y"], w["Ng_z"]], np.float32).view(np.uint32)
        assert got[0] == exp[0], (k, list(out), w)
        if win == w["primID"]:
            assert (got == exp).all(), (k, list(out), w)
    assert hits > 50
    sc.free()


@pytest.mark.parametrize("basis", ["bezier", "bspline", "catmull_rom", "hermite"])
def test_round_cubic_curve_test_equals_oracle(emu, oracle, basis):
    """rt_core.cuh round_cubic_test (RTC_GEOMETRY_TYPE_ROUND_*_CURVE: the sweep intersector with its Newton iteration), host
    instantiation, brute force over all curves: the same winner and bit-identical t / u / Ng as the C oracle's BVH traversal."""
    import ctypes as C
    from embree_b200 import scenes
    from embree_b200.rtc import make_rayhits
    from tests.parity import CUBIC_BASES
    cv, ci, tang = scenes.cubic_hair(90, basis, seed=13, width=0.03)
    sc = oracle.scene([], cubics=[(cv, ci, 1, 0xFFFFFFFF, basis, 4, tang, True)])
    rng = np.random.RandomState(5)
    org = rng.normal(size=(1500, 3)).astype(np.float32)
    org = org / np.linalg.norm(org, axis=1, keepdims=True) * 2.0
    d = (-org + rng.normal(scale=0.35, size=org.shape)).astype(np.float32)
    rays = make_rayhits(org, d)
    rays["tnear"][::7] = 1.1
    want = sc.trace(rays.copy())
    if basis == "hermite":
        k = np.float32(1.0 / 3.0)
        fma = lambda a, b, c: (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)   # noqa: E731
        p0, p1, t0, t1 = cv[ci], cv[ci + 1], tang[ci], tang[ci + 1]
        cps = np.stack([p0, fma(np.full_like(t0, k), t0, p0), fma(np.full_like(t1, -k), t1, p1), p1], 1)
    else:
        cps = np.stack([cv[ci + j] for j in range(4)], 1)
    cps = np.ascontiguousarray(cps, np.float32)
    emu.emu_round_cubic_closest.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_uint, C.c_void_p]
    out = (C.c_float * 6)()
    hits = 0
    for k in range(len(rays)):
        r = rays[k]
        ray = np.array([r["org_x"], r["org_y"], r["org_z"], r["tnear"], r["dir_x"], r["dir_y"], r["dir_z"], r["tfar"]], np.float32)
        win = emu.emu_round_cubic_closest(ray.ctypes.data, cps.ctypes.data, len(ci), 0 if basis == "hermite" else CUBIC_BASES.index(basis), out)
        w = want[k]
        if win < 0:
            assert w["geomID"] == 0xFFFFFFFF, k
            continue
        hits += 1
        got = np.array(list(out), np.float32).view(np.uint32)
        exp = np.array([w["tfar"], w["u"], w["v"], w["Ng_x"], w["Ng_y"], w["Ng_z"]], np.float32).view(np.uint32)
        assert got[0] == exp[0], (k, list(out), w)
        if win == w["primID"]:
            assert (got == exp).all(), (k, list(out), w)
    assert hits > 150
    sc.free()


@pytest.mark.parametrize("n_meshes", [1, 2, 8, 9, 40])
def test_two_level_assembly_equals_single_bvh(emu, oracle, n_meshes):
    """embree_b200/csrc/two_level.h (the host-built top level of two-level dynamic scenes) + the node / record relocation of
    build.cu assemble_scene, on the CPU emulation: `n_meshes` separately built BVH8s assembled under a top level return the hits of
    the oracle's single BVH over all triangles (1 mesh: the root is the mesh's root; <= 8: one top node; more: nested top nodes)."""
    import ctypes as C
    from embree_b200 import scenes
    from embree_b200.rtc import make_rayhits
    rng = np.random.RandomState(3 + n_meshes)
    emu.emu_assemble.restype = C.c_void_p
    emu.emu_assemble.argtypes = [C.c_void_p, C.c_int]
    handles, meshes, keep = [], [], []
    for i in range(n_meshes):
        v, t = scenes.triangle_sphere(int(rng.randint(4, 12)))
        v = (v * np.float32(rng.uniform(0.3, 0.9)) + rng.uniform(-3, 3, 3).astype(np.float32)).astype(np.float32)
        v = np.ascontiguousarray(v); t = np.ascontiguousarray(t, np.uint32)
        keep += [v, t]
        handles.append(emu.emu_build(v.ctypes.data, len(v), t.ctypes.data, len(t), i, 0xFFFFFFFF, 3))
        meshes.append((v, t, i, 0xFFFFFFFF))
    arr = (C.c_void_p * n_meshes)(*handles)
    top = emu.emu_assemble(arr, n_meshes)
    assert top
    org = rng.uniform(-5, 5, (6000, 3)).astype(np.float32)
    d = rng.normal(size=(6000, 3)).astype(np.float32)
    rays = make_rayhits(org, d)
    got = rays.copy()
    emu.emu_trace(top, got.ctypes.data, len(got), 0, None)
    want = oracle.scene(meshes).trace(rays.copy())
    rep = compare_hits(want, got, meshes=meshes)
    assert rep["id_mismatch"] == 0 and rep["hit_miss_disagree"] == 0 and rep["tie"] <= 4 and rep["hits"] > 20, rep
    occ = rays_of(rays)
    emu.emu_trace(top, occ.ctypes.data, len(occ), 1, None)
    assert ((occ["tfar"] == -np.inf) == (want["geomID"] != 0xFFFFFFFF)).all()
    emu.emu_free(top)
    for h in handles:
        emu.emu_free(h)


def point_cloud(n=1500, seed=5):
    """Random point primitives inside the unit cube (centre, radius) + normals, and rays through them: some start inside a
    sphere (back hit), some end before the cloud."""
    rng = np.random.RandomState(seed)
    pv = np.concatenate([rng.uniform(-1, 1, (n, 3)), rng.uniform(0.01, 0.12, (n, 1))], 1).astype(np.float32)
    pn = rng.normal(size=(n, 3)).astype(np.float32)
    m = 4000
    org = rng.normal(size=(m, 3)).astype(np.float32)
    org = org / np.linalg.norm(org, axis=1, keepdims=True) * rng.uniform(0.0, 2.5, (m, 1)).astype(np.float32)
    org[::11] = pv[rng.randint(0, n, len(org[::11])), :3] + np.float32(0.004)     # inside a sphere: only its back side is hit
    d = (rng.uniform(-1, 1, (m, 3)) - org).astype(np.float32) * rng.uniform(0.3, 3, (m, 1)).astype(np.float32)
    rays = make_rayhits(org, d, tnear=1e-3)
    rays["tfar"][::7] = 0.9
    return pv, pn, rays


@pytest.mark.parametrize("kind", ["sphere", "disc", "oriented_disc"])
def test_point_test_equals_oracle(emu, oracle, kind):
    """rt_core.cuh point_test (RTC_GEOMETRY_TYPE_SPHERE_POINT / _DISC_POINT / _ORIENTED_DISC_POINT), host instantiation, brute force
    over all points: the same winner and bit-identical t / Ng as the C oracle's BVH traversal."""
    from tests.parity import POINT_KINDS
    pv, pn, rays = point_cloud()
    sc = oracle.scene([], points=[(pv, kind, pn if kind == "oriented_disc" else None, 2, 0xFFFFFFFF)])
    want = sc.trace(rays.copy())
    emu.emu_point_closest.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    out = np.zeros(6, np.float32)
    hits = 0
    for k in range(len(rays)):
        r = rays[k]
        ray = np.array([r["org_x"], r["org_y"], r["org_z"], r["tnear"], r["dir_x"], r["dir_y"], r["dir_z"], r["tfar"]], np.float32)
        best = emu.emu_point_closest(ray.ctypes.data, pv.ctypes.data, pn.ctypes.data if kind == "oriented_disc" else None, len(pv),
                                     POINT_KINDS.index(kind), out.ctypes.data)
        w = want[k]
        if best < 0:
            assert w["geomID"] == 0xFFFFFFFF, k
            continue
        hits += 1
        assert w["geomID"] == 2 and w["primID"] == best, (k, best, w)
        exp = np.array([w["tfar"], w["u"], w["v"], w["Ng_x"], w["Ng_y"], w["Ng_z"]], np.float32)
        assert (out.view(np.uint32) == exp.view(np.uint32)).all(), (k, out, w)
    assert hits > 1000
    assert np.allclose(sc.bounds(), np.concatenate([(pv[:, :3] - pv[:, 3:]).min(0), (pv[:, :3] + pv[:, 3:]).max(0)]))
    sc.free()


@pytest.mark.parametrize("kind", ["sphere", "disc", "oriented_disc"])
def test_point_test_edge_cases_equal_oracle(emu, oracle, kind):
    """The corners of the point tests' domain (tests/parity.py point_edge_cases): host instantiation of rt_core.cuh point_test, brute
    force, against the C oracle's BVH traversal -- the same winner and bit-identical t / Ng (zero radii, far centres, origins at the
    centre / inside / on the surface, tnear / tfar windows, |dir| from 1e-3 to 1e3, rays parallel to a disc, non-unit normals)."""
    from tests.parity import POINT_KINDS, point_edge_cases
    pv, pn, rays = point_edge_cases()
    sc = oracle.scene([], points=[(pv, kind, pn if kind == "oriented_disc" else None, 2, 0xFFFFFFFF)])
    want = sc.trace(rays.copy())
    sc.free()
    emu.emu_point_closest.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    out = np.zeros(6, np.float32)
    hits = ties = 0
    for k in range(len(rays)):
        r = rays[k]
        ray = np.array([r["org_x"], r["org_y"], r["org_z"], r["tnear"], r["dir_x"], r["dir_y"], r["dir_z"], r["tfar"]], np.float32)
        best = emu.emu_point_closest(ray.ctypes.data, pv.ctypes.data, pn.ctypes.data if kind == "oriented_disc" else None, len(pv),
                                     POINT_KINDS.index(kind), out.ctypes.data)
        w = want[k]
        if best < 0:
            assert w["geomID"] == 0xFFFFFFFF, k
            continue
        hits += 1
        assert w["geomID"] == 2 and np.float32(out[0]).view(np.uint32) == w["tfar"].view(np.uint32), (k, best, out, w)
        if w["primID"] != best:      # two points at exactly the same distance (t = 0 from inside two large spheres): order dependent
            ties += 1
            continue
        exp = np.array([w["tfar"], w["u"], w["v"], w["Ng_x"], w["Ng_y"], w["Ng_z"]], np.float32)
        assert (out.view(np.uint32) == exp.view(np.uint32)).all(), (k, out, w)
    assert hits > 1000 and ties <= 0.02 * hits, (hits, ties)


def _beyond_the_solid(S, ray, gid, prim, t):
    """Does distance t on round linear segment `prim` of geometry `gid` lie outside the segment's float64 solid (tests/curve_exact.py)?"""
    from tests.curve_exact import round_segment_interval
    cv, ci = S["curves"][gid][:2]
    o = np.array([[ray["org_x"][0], ray["org_y"][0], ray["org_z"][0]]], np.float64)
    d = np.array([[ray["dir_x"][0], ray["dir_y"][0], ray["dir_z"][0]]], np.float64)
    t_in, t_out = round_segment_interval(o, d, cv[ci[prim]][None].astype(np.float64), cv[ci[prim] + 1][None].astype(np.float64))
    tol = 1e-3 * float(np.linalg.norm(cv[ci[prim], :3] - o[0]) + cv[ci[prim], 3]) / float(np.linalg.norm(d))
    return not (t_in[0] - tol <= t <= t_out[0] + tol)


def _finite(a):
    return (np.abs(np.nan_to_num(a, nan=np.inf)) < 1.8e18).all(axis=tuple(range(1, a.ndim)))


@pytest.mark.parametrize("kind", CURVE_KINDS)
def test_curve_edge_cases_equal_oracle(emu, oracle, kind):
    """The corners of each curve kind's domain (tests/curve_cases.py curve_edge_cases): host instantiation of rt_core.cuh curve_test /
    flat_curve_test / flat_cubic_test / round_cubic_test, brute force over every valid primitive the ray's mask admits, against the C
    oracle's BVH traversal -- bit-identical t / u / v / Ng; two primitives may swap only at a bit-identical t (a shared joint)."""
    from tests.curve_cases import curve_edge_cases, kind_parts, oracle_scene
    from tests.parity import CUBIC_BASES
    rnd, basis = kind_parts(kind)
    S = curve_edge_cases(kind)
    rays = S["rays"]
    sc = oracle_scene(oracle, S)
    want = sc.trace(rays.copy())
    sc.free()
    sets = []              # (geomID, mask, keep, call(ray8) -> winning position in keep[-1] or -1; the hit in `out`)
    out = np.zeros(6, np.float32)
    if basis is None:
        emu.emu_linear_curve_closest.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        for (cv, ci, cf, gid, mask, flat) in S["curves"]:
            if cf is None:                                   # library-derived flags: neighbours are consecutive segments
                cf = np.zeros(len(ci), np.uint8)
                cf[:-1] |= np.where(ci[1:] == ci[:-1] + 1, 2, 0).astype(np.uint8)
                cf[1:] |= (cf[:-1] >> 1) & 1
            ok = np.nonzero(_finite(cv[ci]) & _finite(cv[ci + 1]) & (np.minimum(cv[ci, 3], cv[ci + 1, 3]) >= 0))[0]
            keep = (np.ascontiguousarray(cv, np.float32), np.ascontiguousarray(ci[ok], np.uint32), np.ascontiguousarray(cf[ok], np.uint8), ok)
            sets.append((gid, mask, keep, lambda ray, k=keep, fl=flat: emu.emu_linear_curve_closest(
                ray.ctypes.data, k[0].ctypes.data, k[1].ctypes.data, k[2].ctypes.data, len(k[1]), int(fl), out.ctypes.data)))
    else:
        emu.emu_flat_cubic_closest.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_uint, C.c_int, C.c_void_p]
        emu.emu_round_cubic_closest.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_uint, C.c_void_p]
        for (cv, ci, gid, mask, b, tess, tg, _r) in S["cubics"]:
            if b == "hermite":    # the conversion HermiteCurveT does (hermite_curve.h:19-20), with the same fused operations
                k3 = np.float32(1.0 / 3.0)
                fma = lambda a, x, c: (a.astype(np.float64) * x.astype(np.float64) + c.astype(np.float64)).astype(np.float32)   # noqa: E731
                p0, p1, t0, t1 = cv[ci], cv[ci + 1], tg[ci], tg[ci + 1]
                with np.errstate(invalid="ignore", over="ignore"):
                    cps = np.stack([p0, fma(np.full_like(t0, k3), t0, p0), fma(np.full_like(t1, -k3), t1, p1), p1], 1)
                ok = _finite(cps) & _finite(np.stack([p0, p1, t0, t1], 1))
            else:
                cps = np.stack([cv[ci + j] for j in range(4)], 1)
                ok = _finite(cps)
            ok = np.nonzero(ok)[0]
            keep = (np.ascontiguousarray(cps[ok], np.float32), ok)
            bi = 0 if b == "hermite" else CUBIC_BASES.index(b)
            if rnd:
                call = lambda ray, k=keep, bi=bi: emu.emu_round_cubic_closest(ray.ctypes.data, k[0].ctypes.data, len(k[0]), bi, out.ctypes.data)   # noqa: E731
            else:
                call = lambda ray, k=keep, bi=bi, n=tess: emu.emu_flat_cubic_closest(ray.ctypes.data, k[0].ctypes.data, len(k[0]), bi, n, out.ctypes.data)   # noqa: E731
            sets.append((gid, mask, keep, call))
    hits = ties = spills = 0
    for k in range(len(rays)):
        r = rays[k]
        ray = np.array([r["org_x"], r["org_y"], r["org_z"], r["tnear"], r["dir_x"], r["dir_y"], r["dir_z"], r["tfar"]], np.float32)
        best = None
        for (gid, mask, keep, call) in sets:
            if not (int(r["mask"]) & mask):
                continue
            w = call(ray)
            if w >= 0:
                best = (gid, int(keep[-1][w]), out.copy())
                ray[7] = out[0]
        w = want[k]
        if (best is None) != (w["geomID"] == 0xFFFFFFFF) or (best is not None and best[2].view(np.uint32)[0] != w["tfar"].view(np.uint32)):
            # a round linear cone accepts hits a little beyond its end sphere (the band test y > -ulp takes an absolute ulp, wide at a
            # 1e-3 scale), outside the segment's solid and box: whether a traversal offers that segment depends on its leaf boxes
            near = min([x for x in ((best[0], best[1], float(best[2][0])) if best else None,
                                    (int(w["geomID"]), int(w["primID"]), float(w["tfar"])) if w["geomID"] != 0xFFFFFFFF else None) if x],
                       key=lambda x: x[2])
            assert kind == "round_linear" and _beyond_the_solid(S, rays[k:k + 1], *near), (k, best, w)
            spills += 1
            continue
        if best is None:
            continue
        hits += 1
        exp = np.array([w["tfar"], w["u"], w["v"], w["Ng_x"], w["Ng_y"], w["Ng_z"]], np.float32)
        assert w["geomID"] == best[0], (k, best, w)
        if w["primID"] != best[1]:          # the same distance on two primitives: the joint of two segments of one strand
            ties += 1
            continue
        assert (best[2].view(np.uint32) == exp.view(np.uint32)).all(), (k, best, w)
    print(kind, dict(rays=len(rays), hits=hits, ties=ties, beyond_the_solid=spills))
    assert hits > 900 and ties <= 0.02 * hits and spills <= 0.01 * len(rays), (hits, ties, spills)
