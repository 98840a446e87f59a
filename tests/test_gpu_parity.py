"""GPU parity tests: every call goes through the C-ABI of embree_b200/csrc/libembree4_b200.so (no oracle, no CPU code on
the product path) and is compared with the golden vectors of the unmodified reference, the C oracle and -- when
oracle/_ref travelled to the box -- the reference library run side by side.  Structure follows the reference's
verify suite (tutorials/verify/verify.cpp): the same RTCRayHit[] is fed through every entry point
(rtcore_helpers.h:701-787 IntersectWithMode) and occluded is cross-checked against intersect (:787-790).

Bar (BASELINE.json): primID / geomID / instID bit-exact, t/u/v within 1e-4 relative."""
import ctypes as C

import numpy as np
import pytest

from embree_b200 import scenes
from embree_b200.rtc import (RTCBounds, RTC_BUILD_QUALITY_LOW, RTC_BUILD_QUALITY_MEDIUM, RTC_FORMAT_FLOAT3, RTC_FORMAT_UINT3,
                             RTC_BUFFER_TYPE_INDEX, RTC_BUFFER_TYPE_VERTEX, RTC_GEOMETRY_TYPE_TRIANGLE, RTC_GEOMETRY_TYPE_INSTANCE, RTC_FORMAT_FLOAT3X4_ROW_MAJOR,
                             RTC_FORMAT_FLOAT3X4_COLUMN_MAJOR, RTC_FORMAT_FLOAT4X4_COLUMN_MAJOR, aligned_empty,
                             make_rayhits, rays_of, to_packets, from_packets, _ptr)
from tests.conftest import GOLDEN, GOLDEN_QUADS, load_golden, load_golden_instances
from tests.parity import compare_hits, explain_hit_miss, reference_outputs

pytestmark = pytest.mark.gpu
TOL = 1e-4
MODES = ["1", "4", "8", "16", "1M", "4M", "8M", "16M"]


def build_scene(lib, dev, meshes, quality=RTC_BUILD_QUALITY_MEDIUM, flags=0):
    sc = lib.rtcNewScene(dev)
    lib.rtcSetSceneBuildQuality(sc, quality)
    if flags:
        lib.rtcSetSceneFlags(sc, flags)
    keep = []
    for (v, t, gid, mask) in meshes:
        add = lib.add_quad_mesh if np.asarray(t).shape[1] == 4 else lib.add_triangle_mesh
        _, k = add(dev, sc, v, t, mask=mask, geom_id=gid)
        keep.append(k)
    lib.rtcCommitScene(sc)
    lib.check(dev)
    return sc, keep


def assert_parity(want, got, allow_ties=0):
    rep = compare_hits(want, got, TOL)
    assert rep["id_mismatch"] == 0 and rep["hit_miss_disagree"] == 0 and rep["tie"] <= allow_ties, rep
    assert rep["max_rel_t"] <= TOL and rep["max_abs_uv"] <= TOL and rep["miss_untouched"], rep
    return rep


@pytest.mark.parametrize("robust", [False, True])
@pytest.mark.parametrize("quality", [RTC_BUILD_QUALITY_LOW, RTC_BUILD_QUALITY_MEDIUM])
@pytest.mark.parametrize("name", GOLDEN)
def test_golden_all_entry_points(b200, name, quality, robust):
    """robust=True: RTC_SCENE_FLAG_ROBUST (Triangle4v + Pluecker in the reference, scene.cpp:181-188)."""
    lib, dev = b200
    meshes, rin, want_i, want_o, bounds = load_golden(name, robust)
    sc, keep = build_scene(lib, dev, meshes, quality, flags=4 if robust else 0)
    for mode in MODES:
        got = lib.intersect(sc, rin.copy(), mode)
        rep = assert_parity(want_i, got)
        assert rep["ng_bit_exact"], (mode, rep)
        occ = lib.occluded(sc, rays_of(rin), mode)
        assert (occ["tfar"].view(np.uint32) == want_o["tfar"].view(np.uint32)).all(), mode
    b = RTCBounds()
    lib.rtcGetSceneBounds(sc, C.byref(b))
    assert np.array_equal(np.array([b.lower_x, b.lower_y, b.lower_z, b.upper_x, b.upper_y, b.upper_z], np.float32), bounds)
    lib.check(dev)
    lib.rtcReleaseScene(sc)


def test_triangle_hit_kat(b200):
    """TriangleHitTest, verify.cpp:2462-2547."""
    lib, dev = b200
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32)
    t = np.array([[0, 1, 2]], np.uint32)
    sc, keep = build_scene(lib, dev, [(v, t, 0, 0xFFFFFFFF)])
    u0, v0 = np.meshgrid((np.arange(16) + 0.5) / 16 * 0.45, (np.arange(16) + 0.5) / 16 * 0.45)
    org = np.stack([u0.ravel(), v0.ravel(), -np.ones(256)], 1).astype(np.float32)
    for mode in MODES:
        out = lib.intersect(sc, make_rayhits(org, np.tile([[0, 0, 1]], (256, 1))), mode)
        ulp = 16 * np.finfo(np.float32).eps
        assert (out["geomID"] == 0).all() and (out["primID"] == 0).all() and (out["instID"] == 0xFFFFFFFF).all()
        assert np.abs(out["u"] - org[:, 0]).max() <= ulp and np.abs(out["v"] - org[:, 1]).max() <= ulp
        assert np.abs(out["tfar"] - 1.0).max() <= ulp
        assert (out["Ng_x"] == 0).all() and (out["Ng_y"] == 0).all() and (out["Ng_z"] == 1).all()
    lib.rtcReleaseScene(sc)


def test_inactive_lanes_untouched(b200):
    """InactiveRaysTest, verify.cpp:3553-3609: lanes with valid == 0 come back bit-identical."""
    lib, dev = b200
    v, t = scenes.triangle_sphere(16)
    sc, keep = build_scene(lib, dev, [(v, t, 0, 0xFFFFFFFF)])
    rays = scenes.as_numpy_rayhits(scenes.incoherent_rays_reference(256))
    a = lib.args()
    for K in (4, 8, 16):
        p, valid = to_packets(rays.copy(), K)
        rng = np.random.RandomState(K)
        valid[:] = np.where(rng.rand(len(valid)) < 0.5, -1, 0)
        before = p.copy()
        fn = getattr(lib, f"rtcIntersect{K}")
        for i in range(len(p)):
            fn(C.c_void_p(valid.ctypes.data + 4 * K * i), sc, C.c_void_p(p.ctypes.data + p.dtype.itemsize * i), C.byref(a))
        after = from_packets(p, len(rays))
        orig = from_packets(before, len(rays))
        inactive = valid[:len(rays)] == 0
        assert (after.view(np.uint8).reshape(-1, 96)[inactive] == orig.view(np.uint8).reshape(-1, 96)[inactive]).all()
        assert (after["geomID"][~inactive] == 0).all()
        # batched variant
        p2 = before.copy()
        lib.rtcb200IntersectNM(_ptr(valid), sc, _ptr(p2), K, len(p2), C.byref(a))
        assert (p2.view(np.uint8) == p.view(np.uint8)).all()
    lib.check(dev)
    lib.rtcReleaseScene(sc)


def test_ray_masks(b200):
    """RayMasksTest, verify.cpp:2626-2692: geometry i has mask 1<<i; a ray sees it iff (mask & ray.mask) != 0."""
    lib, dev = b200
    meshes = []
    for i in range(4):
        v, t = scenes.triangle_plane((-1, -1, 1.0 + i), (2, 0, 0), (0, 2, 0), 2, 2)
        meshes.append((v, t, i, 1 << i))
    sc, keep = build_scene(lib, dev, meshes)
    org = np.tile([[0.1, 0.2, 0.0]], (16, 1)).astype(np.float32)
    d = np.tile([[0, 0, 1]], (16, 1)).astype(np.float32)
    r = make_rayhits(org, d)
    r["mask"] = np.arange(16, dtype=np.uint32)
    for mode in ("1", "16", "1M"):
        out = lib.intersect(sc, r.copy(), mode)
        for m in range(16):
            want = next((i for i in range(4) if m & (1 << i)), None)
            if want is None:
                assert out["geomID"][m] == 0xFFFFFFFF
            else:
                assert out["geomID"][m] == want and abs(out["tfar"][m] - (1.0 + want)) < 1e-6
        occ = lib.occluded(sc, rays_of(r), mode)
        assert ((occ["tfar"] == -np.inf) == (np.arange(16) != 0)).all()
    lib.rtcReleaseScene(sc)


def test_empty_scene_and_garbage_geometry(b200):
    """EmptySceneTest (verify.cpp:1054), GarbageGeometryTest (:1915): nothing to hit, no crash, invalid triangles dropped."""
    lib, dev = b200
    sc = lib.rtcNewScene(dev)
    lib.rtcCommitScene(sc)
    lib.check(dev)
    out = lib.intersect(sc, make_rayhits([[0, 0, -1]], [[0, 0, 1]]), "1")
    assert out["geomID"][0] == 0xFFFFFFFF and np.isinf(out["tfar"][0])
    lib.rtcReleaseScene(sc)
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [np.nan, 0, 0], [2e18, 0, 0], [np.inf, 1, 1]], np.float32)
    t = np.array([[0, 1, 2], [0, 1, 3], [0, 1, 4], [0, 1, 77], [5, 1, 2]], np.uint32)
    sc, keep = build_scene(lib, dev, [(v, t, 0, 0xFFFFFFFF)])
    assert lib.scene_stats(sc).num_triangles == 1
    out = lib.intersect(sc, make_rayhits([[0.2, 0.2, -1], [5, 5, -1]], [[0, 0, 1], [0, 0, 1]]), "1M")
    assert out["primID"][0] == 0 and out["geomID"][1] == 0xFFFFFFFF
    lib.rtcReleaseScene(sc)
    rng = np.random.RandomState(0)
    v = rng.uniform(-1e30, 1e30, (300, 3)).astype(np.float32)
    v[::7] = np.nan
    t = rng.randint(0, 400, (500, 3)).astype(np.uint32)
    sc, keep = build_scene(lib, dev, [(v, t, 0, 0xFFFFFFFF)])
    lib.intersect(sc, scenes.as_numpy_rayhits(scenes.incoherent_rays_reference(1000)), "1M")
    lib.check(dev)
    lib.rtcReleaseScene(sc)


def test_nan_inf_rays_terminate(b200):
    lib, dev = b200
    v, t = scenes.triangle_sphere(16)
    sc, keep = build_scene(lib, dev, [(v, t, 0, 0xFFFFFFFF)])
    org, d = [], []
    for b in (np.nan, np.inf, -np.inf):
        org += [[b, 0, 0], [0, 0, 0], [0, b, 0]]
        d += [[0, 0, 1], [b, 0, 1], [1, b, b]]
    lib.intersect(sc, make_rayhits(np.array(org, np.float32), np.array(d, np.float32)), "1M")
    lib.check(dev)
    lib.rtcReleaseScene(sc)


def test_buffer_stride_and_owned_buffers(b200):
    """BufferStrideTest (verify.cpp:915): strides != 12, byte offsets, rtcSetNewGeometryBuffer / rtcNewBuffer."""
    lib, dev = b200
    v, t = scenes.triangle_sphere(12)
    rays = scenes.as_numpy_rayhits(scenes.incoherent_rays_reference(2000))
    sc0, k0 = build_scene(lib, dev, [(v, t, 0, 0xFFFFFFFF)])
    want = lib.intersect(sc0, rays.copy(), "1M")
    # (a) shared buffers with stride 16 / 20 and a byte offset
    vb = np.zeros((len(v) + 2, 4), np.float32)
    vb[1:len(v) + 1, :3] = v
    ib = np.zeros((len(t), 5), np.uint32)
    ib[:, 1:4] = t
    g = lib.rtcNewGeometry(dev, RTC_GEOMETRY_TYPE_TRIANGLE)
    lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, _ptr(vb), 16, 16, len(v))
    lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT3, _ptr(ib), 4, 20, len(t))
    lib.rtcSetGeometryMask(g, 0xFFFFFFFF)
    lib.rtcCommitGeometry(g)
    sc = lib.rtcNewScene(dev)
    lib.rtcAttachGeometry(sc, g)
    lib.rtcReleaseGeometry(g)
    lib.rtcCommitScene(sc)
    lib.check(dev)
    got = lib.intersect(sc, rays.copy(), "1M")
    assert (got.view(np.uint8) == want.view(np.uint8)).all()
    lib.rtcReleaseScene(sc)
    # (b) geometry-owned buffers + an rtcNewBuffer-backed index buffer
    g = lib.rtcNewGeometry(dev, RTC_GEOMETRY_TYPE_TRIANGLE)
    pv = lib.rtcSetNewGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, 12, len(v))
    C.memmove(pv, v.ctypes.data, v.nbytes)
    buf = lib.rtcNewBuffer(dev, t.nbytes)
    C.memmove(lib.rtcGetBufferData(buf), t.ctypes.data, t.nbytes)
    lib.rtcSetGeometryBuffer(g, RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT3, buf, 0, 12, len(t))
    lib.rtcReleaseBuffer(buf)
    lib.rtcSetGeometryMask(g, 0xFFFFFFFF)
    lib.rtcCommitGeometry(g)
    sc = lib.rtcNewScene(dev)
    lib.rtcAttachGeometry(sc, g)
    lib.rtcReleaseGeometry(g)
    lib.rtcCommitScene(sc)
    lib.check(dev)
    got = lib.intersect(sc, rays.copy(), "1M")
    assert (got.view(np.uint8) == want.view(np.uint8)).all()
    lib.rtcReleaseScene(sc)
    lib.rtcReleaseScene(sc0)


def test_commit_state_machine_and_errors(b200):
    """geometry.cpp:97-135, scene_verify.cpp:11-22, rtcore.cpp:405: error codes of the commit protocol."""
    lib, dev = b200
    assert lib.rtcGetDeviceError(dev) == 0
    sc = lib.rtcNewScene(dev)
    b = RTCBounds()
    lib.rtcGetSceneBounds(sc, C.byref(b))
    assert lib.rtcGetDeviceError(dev) == 3          # scene not committed
    assert lib.rtcGetDeviceError(dev) == 0          # reading clears the slot
    r = make_rayhits([[0, 0, -1]], [[0, 0, 1]])
    lib.rtcIntersect1(sc, _ptr(r), None)
    assert lib.rtcGetDeviceError(dev) == 3          # intersecting an uncommitted scene (scene.cpp:36,65)
    v, t = scenes.triangle_sphere(6)
    g = lib.rtcNewGeometry(dev, RTC_GEOMETRY_TYPE_TRIANGLE)
    vpad = np.zeros(v.size + 4, np.float32)
    vpad[:v.size] = v.ravel()
    lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, _ptr(vpad), 0, 12, len(v))
    lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT3, _ptr(t), 0, 12, len(t))
    gid = lib.rtcAttachGeometry(sc, g)
    assert gid == 0
    lib.rtcCommitScene(sc)
    assert lib.rtcGetDeviceError(dev) == 3          # geometry not committed
    lib.rtcCommitGeometry(g)
    lib.rtcCommitScene(sc)
    assert lib.rtcGetDeviceError(dev) == 0
    out = lib.intersect(sc, make_rayhits([[0, 0, 0]], [[0, 0, 1]]), "1")
    assert out["geomID"][0] == 0                    # default geometry mask is 1 (geometry.cpp:48), ray mask -1 -> visible
    r2 = make_rayhits([[0, 0, 0]], [[0, 0, 1]], mask=0x2)
    assert lib.intersect(sc, r2, "1")["geomID"][0] == 0xFFFFFFFF
    # wrong formats / slots (scene_triangle_mesh.cpp:35-80)
    lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_UINT3, _ptr(vpad), 0, 12, len(v))
    assert lib.rtcGetDeviceError(dev) == 3
    lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_INDEX, 1, RTC_FORMAT_UINT3, _ptr(t), 0, 12, len(t))
    assert lib.rtcGetDeviceError(dev) == 2
    lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, _ptr(vpad), 2, 12, len(v))
    assert lib.rtcGetDeviceError(dev) == 3          # not 4-byte aligned
    assert not lib.rtcNewGeometry(dev, 8)           # subdivision surfaces unsupported
    assert lib.rtcGetDeviceError(dev) == 3
    # disable / enable / detach
    lib.rtcDisableGeometry(g)
    lib.rtcCommitScene(sc)
    assert lib.intersect(sc, make_rayhits([[0, 0, 0]], [[0, 0, 1]]), "1")["geomID"][0] == 0xFFFFFFFF
    lib.rtcEnableGeometry(g)
    lib.rtcCommitScene(sc)
    assert lib.intersect(sc, make_rayhits([[0, 0, 0]], [[0, 0, 1]]), "1")["geomID"][0] == 0
    lib.rtcDetachGeometry(sc, 0)
    lib.rtcCommitScene(sc)
    assert lib.intersect(sc, make_rayhits([[0, 0, 0]], [[0, 0, 1]]), "1")["geomID"][0] == 0xFFFFFFFF
    assert lib.rtcGetDeviceError(dev) == 0
    lib.rtcReleaseGeometry(g)
    lib.rtcReleaseScene(sc)


@pytest.mark.parametrize("robust", [False, True])
@pytest.mark.parametrize("quality", [RTC_BUILD_QUALITY_LOW, RTC_BUILD_QUALITY_MEDIUM])
@pytest.mark.parametrize("name", GOLDEN_QUADS)
def test_quads_golden_all_entry_points(b200, name, quality, robust):
    """RTC_GEOMETRY_TYPE_QUAD next to triangle meshes against the reference's own outputs (quad_intersector_moeller.h,
    quad_intersector_pluecker.h): ids exact, t/u/v within 1e-4, Ng bit-exact away from the quad diagonal (ON the shared
    diagonal the reference's 8-wide min-t selection between the two halves is decided by rounding noise)."""
    lib, dev = b200
    meshes, rin, want_i, want_o, bounds = load_golden(name, robust)
    sc, keep = build_scene(lib, dev, meshes, quality, flags=4 if robust else 0)
    for mode in MODES:
        got = lib.intersect(sc, rin.copy(), mode)
        assert_parity(want_i, got)
        hit = want_i["geomID"] != 0xFFFFFFFF
        off_diag = hit & (np.abs(want_i["u"] + want_i["v"] - 1.0) > 1e-4)
        for f in ("Ng_x", "Ng_y", "Ng_z"):
            assert (want_i[f].view(np.uint32) == got[f].view(np.uint32))[off_diag].all(), (mode, f)
        occ = lib.occluded(sc, rays_of(rin), mode)
        assert (occ["tfar"].view(np.uint32) == want_o["tfar"].view(np.uint32)).all(), mode
    b = RTCBounds()
    lib.rtcGetSceneBounds(sc, C.byref(b))
    assert np.array_equal(np.array([b.lower_x, b.lower_y, b.lower_z, b.upper_x, b.upper_y, b.upper_z], np.float32), bounds)
    lib.rtcReleaseScene(sc)


def test_quads_large_vs_oracle(b200, oracle):
    """1M non-planar quads (2M half records) + an instanced quad scene against the C oracle: invalid quads dropped
    whole, quad primIDs reported, instancing of quad meshes."""
    lib, dev = b200
    v, q = scenes.quad_terrain(1000, seed=9)
    q = q.copy()
    q[5] = (0, 1, 2, 0xFFFFFFF0)        # out-of-range index: the WHOLE quad is invalid (scene_quad_mesh.h:186-203)
    v = v.copy()
    v[int(q[77, 2])] = np.nan            # NaN vertex: every quad that references it is dropped
    sc, keep = build_scene(lib, dev, [(v, q, 0, 0xFFFFFFFF)])
    rng = np.random.RandomState(3)
    org = rng.uniform(-1, 1, (300000, 3)).astype(np.float32)
    org[:, 1] = 0.5
    d = rng.normal(size=(300000, 3)).astype(np.float32)
    d[:, 1] = -np.abs(d[:, 1])
    rays = make_rayhits(org, d)
    got = lib.intersect(sc, rays.copy(), "1M")
    osc = oracle.scene([(v, q, 0, 0xFFFFFFFF)])
    want = osc.trace(rays.copy(), nthreads=16)
    rep = compare_hits(want, got, TOL, meshes=[(v, q, 0, 0xFFFFFFFF)])
    assert rep["hits"] > 100000 and rep["id_mismatch"] == 0, rep       # ties: same t (4 ulp) on a shared edge / vertex only
    assert rep["max_rel_t"] <= TOL and rep["max_abs_uv"] <= TOL, rep
    # hit/miss disagreements are explained ray by ray: the GPU never loses a hit, and each extra GPU hit is accepted by
    # the reference arithmetic on that quad alone (the reference's unpadded box test culled it in the full scene)
    lost, unexplained = explain_hit_miss(oracle, rays, want, got, lambda g_, p_, i_: oracle.scene([(v, q[p_:p_ + 1], 0, 0xFFFFFFFF)]))
    assert lost == 0 and unexplained == 0, (rep, lost, unexplained)
    assert got["primID"][got["geomID"] == 0].max() < len(q)
    # the same quad mesh seen through two instances
    top = lib.rtcNewScene(dev)
    xf = [np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], np.float32), np.array([0.5, 0, 0, 0, 0.5, 0, 0, 0, 0.5, 0, 0.3, 0], np.float32)]
    for m in xf:
        lib.add_instance(dev, top, sc, m, mask=0xFFFFFFFF)
    lib.rtcCommitScene(top)
    lib.check(dev)
    got2 = lib.intersect(top, rays[:50000].copy(), "1M")
    otop = oracle.scene([], instances=[(osc, m, i, 0xFFFFFFFF) for i, m in enumerate(xf)])
    want2 = otop.trace(rays[:50000].copy(), nthreads=16)
    rep2 = compare_hits(want2, got2, TOL)
    assert rep2["id_mismatch"] == 0, rep2

    def one_quad_instanced(g_, p_, i_):
        c = oracle.scene([(v, q[p_:p_ + 1], 0, 0xFFFFFFFF)])
        return oracle.scene([], instances=[(c, xf[i_], i_, 0xFFFFFFFF)])
    lost2, unexplained2 = explain_hit_miss(oracle, rays[:50000], want2, got2, one_quad_instanced)
    assert lost2 == 0 and unexplained2 == 0, (rep2, lost2, unexplained2)
    assert (got2["instID"][got2["geomID"] != 0xFFFFFFFF] <= 1).all() and (got2["instID"] == 1).sum() > 1000
    otop.free()
    osc.free()
    lib.rtcReleaseScene(top)
    lib.rtcReleaseScene(sc)


def build_instanced(lib, dev, g, quality=RTC_BUILD_QUALITY_MEDIUM):
    child, keep = build_scene(lib, dev, g["child"], quality)
    top = lib.rtcNewScene(dev)
    lib.rtcSetSceneBuildQuality(top, quality)
    for (v, t, gid, mask) in g["top"]:
        keep.append(lib.add_triangle_mesh(dev, top, v, t, mask=mask, geom_id=gid)[1])
    for i, m in enumerate(g["xfms"]):
        lib.add_instance(dev, top, child, m, mask=int(g["inst_masks"][i]), geom_id=g["first_inst"] + i)
    lib.rtcCommitScene(top)
    lib.check(dev)
    return top, child, keep


@pytest.mark.parametrize("quality", [RTC_BUILD_QUALITY_LOW, RTC_BUILD_QUALITY_MEDIUM])
def test_instances_golden_all_entry_points(b200, quality):
    """Single-level instancing (tutorials/instanced_geometry, instance_intersector.cpp:15-67) against the reference's own
    outputs: geomID / primID / instID / instPrimID exact, object-space Ng bit-exact, t/u/v within 1e-4 (the device
    intersects the world-space triangle, the reference the object-space one with a transformed ray)."""
    lib, dev = b200
    g = load_golden_instances()
    top, child, keep = build_instanced(lib, dev, g, quality)
    want = g["intersect_out"]
    for mode in MODES:
        got = lib.intersect(top, g["rays_in"].copy(), mode)
        rep = assert_parity(want, got)
        assert rep["ng_bit_exact"], (mode, rep)
        assert (got["instPrimID"] == want["instPrimID"]).all(), mode
        occ = lib.occluded(top, rays_of(g["rays_in"]), mode)
        assert (occ["tfar"].view(np.uint32) == g["occluded_out"]["tfar"].view(np.uint32)).all(), mode
    b = RTCBounds()
    lib.rtcGetSceneBounds(top, C.byref(b))
    assert np.array_equal(np.array([b.lower_x, b.lower_y, b.lower_z, b.upper_x, b.upper_y, b.upper_z], np.float32), g["bounds"])
    lib.rtcReleaseScene(top)
    lib.rtcReleaseScene(child)


def test_instances_many_vs_oracle(b200, oracle):
    """400 instances of a 3.2k-triangle mesh (1.3M flattened triangles) + 200k random rays against the C oracle's
    two-level traversal; transforms include mirrored (negative determinant) and strongly anisotropic ones."""
    lib, dev = b200
    rng = np.random.RandomState(21)
    v, t = scenes.triangle_sphere(40)
    xf = []
    for i in range(400):
        q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        sc = rng.uniform(0.3, 2.0, 3) * (1 if i % 5 else -1)
        m = (q * sc).astype(np.float32)
        xf.append(np.concatenate([m.T.reshape(-1), rng.uniform(-20, 20, 3)]).astype(np.float32))
    g = dict(child=[(v, t, 0, 0xFFFFFFFF)], top=[], xfms=np.stack(xf), inst_masks=np.full(400, 0xFFFFFFFF, np.uint32), first_inst=0)
    top, child, keep = build_instanced(lib, dev, g)
    org = rng.uniform(-25, 25, (200000, 3)).astype(np.float32)
    d = rng.normal(size=(200000, 3)).astype(np.float32)
    rays = make_rayhits(org, d)
    got = lib.intersect(top, rays.copy(), "1M")
    oc = oracle.scene(g["child"])
    ot = oracle.scene([], instances=[(oc, m, i, 0xFFFFFFFF) for i, m in enumerate(xf)])
    want = ot.trace(rays.copy(), nthreads=16)
    rep = compare_hits(want, got, TOL)
    assert rep["hits"] > 20000, rep
    assert rep["id_mismatch"] == 0, rep   # overlapping instances: hits at the same t (4 ulp) are order-dependent ties

    def one_tri_instanced(g_, p_, i_):
        c = oracle.scene([(v, t[p_:p_ + 1], 0, 0xFFFFFFFF)])
        return oracle.scene([], instances=[(c, xf[i_], i_, 0xFFFFFFFF)])
    lost, unexplained = explain_hit_miss(oracle, rays, want, got, one_tri_instanced)
    assert lost == 0 and unexplained == 0, (rep, lost, unexplained)
    assert rep["max_rel_t"] <= TOL and rep["max_abs_uv"] <= TOL and rep["ng_bit_exact"], rep
    occ = lib.occluded(top, rays_of(rays), "1M")
    assert ((occ["tfar"] == -np.inf) != (got["geomID"] != 0xFFFFFFFF)).sum() == 0
    ot.free()
    oc.free()
    lib.rtcReleaseScene(top)
    lib.rtcReleaseScene(child)


def test_instance_api_and_errors(b200):
    """rtcSetGeometryTransform formats (rtcore.cpp:1408-1439), get/set round trip, commit protocol of instances."""
    lib, dev = b200
    v, t = scenes.triangle_sphere(8)
    child, keep = build_scene(lib, dev, [(v, t, 0, 0xFFFFFFFF)])
    g = lib.rtcNewGeometry(dev, RTC_GEOMETRY_TYPE_INSTANCE)
    top = lib.rtcNewScene(dev)
    lib.rtcAttachGeometry(top, g)
    lib.rtcCommitGeometry(g)
    lib.rtcCommitScene(top)
    assert lib.rtcGetDeviceError(dev) == 3                      # no instanced scene set
    lib.rtcSetGeometryInstancedScene(g, child)
    col = np.array([2, 0, 0, 0, 2, 0, 0, 0, 2, 5, 6, 7], np.float32)   # scale 2, translate (5,6,7)
    row = np.array([2, 0, 0, 5, 0, 2, 0, 6, 0, 0, 2, 7], np.float32)
    c44 = np.array([2, 0, 0, 0, 0, 2, 0, 0, 0, 0, 2, 0, 5, 6, 7, 1], np.float32)
    for fmt, m in ((RTC_FORMAT_FLOAT3X4_COLUMN_MAJOR, col), (RTC_FORMAT_FLOAT3X4_ROW_MAJOR, row), (RTC_FORMAT_FLOAT4X4_COLUMN_MAJOR, c44)):
        lib.rtcSetGeometryTransform(g, 0, fmt, _ptr(m))
        lib.rtcCommitGeometry(g)
        lib.rtcCommitScene(top)
        lib.check(dev)
        out = lib.intersect(top, make_rayhits([[5, 6, 0]], [[0, 0, 1]]), "1")
        assert out["geomID"][0] == 0 and out["instID"][0] == 0 and abs(out["tfar"][0] - 5.0) < 1e-5, (fmt, out)
        for f2, m2 in ((RTC_FORMAT_FLOAT3X4_COLUMN_MAJOR, col), (RTC_FORMAT_FLOAT3X4_ROW_MAJOR, row), (RTC_FORMAT_FLOAT4X4_COLUMN_MAJOR, c44)):
            back = np.zeros(len(m2), np.float32)
            lib.rtcGetGeometryTransform(g, 0.0, f2, _ptr(back))
            assert np.array_equal(back, m2), (fmt, f2, back)
    lib.rtcSetGeometryTransform(g, 0, RTC_FORMAT_FLOAT3, _ptr(col))
    assert lib.rtcGetDeviceError(dev) == 3                      # invalid matrix format
    lib.rtcSetGeometryTransform(g, 1, RTC_FORMAT_FLOAT3X4_COLUMN_MAJOR, _ptr(col))
    assert lib.rtcGetDeviceError(dev) == 3                      # motion blur time steps are out of scope
    mesh = lib.rtcNewGeometry(dev, RTC_GEOMETRY_TYPE_TRIANGLE)
    lib.rtcSetGeometryInstancedScene(mesh, child)
    assert lib.rtcGetDeviceError(dev) == 3                      # not an instance
    lib.rtcReleaseGeometry(mesh)
    # moving the instance = set transform + commit geometry + commit scene (dynamic_scene / instanced_geometry tutorials)
    col[9:] = (0, 0, 10)
    lib.rtcSetGeometryTransform(g, 0, RTC_FORMAT_FLOAT3X4_COLUMN_MAJOR, _ptr(col))
    lib.rtcCommitGeometry(g)
    lib.rtcCommitScene(top)
    out = lib.intersect(top, make_rayhits([[0, 0, 0]], [[0, 0, 1]]), "1")
    assert abs(out["tfar"][0] - 8.0) < 1e-5 and out["instID"][0] == 0
    # instance mask and ray mask (instance_intersector.cpp:19-23)
    lib.rtcSetGeometryMask(g, 0x4)
    lib.rtcCommitGeometry(g)
    lib.rtcCommitScene(top)
    assert lib.intersect(top, make_rayhits([[0, 0, 0]], [[0, 0, 1]], mask=0x3), "1")["geomID"][0] == 0xFFFFFFFF
    assert lib.intersect(top, make_rayhits([[0, 0, 0]], [[0, 0, 1]], mask=0x4), "1")["geomID"][0] == 0
    # two-level nesting is rejected (RTC_MAX_INSTANCE_LEVEL_COUNT == 1)
    top2 = lib.rtcNewScene(dev)
    lib.add_instance(dev, top2, top, col)
    lib.rtcCommitScene(top2)
    assert lib.rtcGetDeviceError(dev) == 3
    # the instanced scene stays alive through the instance's reference
    lib.rtcReleaseScene(child)
    assert lib.intersect(top, make_rayhits([[0, 0, 0]], [[0, 0, 1]], mask=0x4), "1")["geomID"][0] == 0
    lib.check(dev)
    lib.rtcReleaseGeometry(g)
    lib.rtcReleaseScene(top)
    lib.rtcReleaseScene(top2)


def test_child_scene_recommit_reaches_the_instance(b200):
    """Instances are flattened into the top-level BVH at commit; the reference traverses the child BVH live, so there
    `rtcCommitScene(child); rtcCommitScene(top)` shows the edited child.  Same protocol, same result here."""
    lib, dev = b200
    v, t = scenes.triangle_sphere(10)
    vpad = np.zeros(v.size + 4, np.float32)
    vpad[:v.size] = v.ravel()
    g = lib.rtcNewGeometry(dev, RTC_GEOMETRY_TYPE_TRIANGLE)
    lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, _ptr(vpad), 0, 12, len(v))
    lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT3, _ptr(t), 0, 12, len(t))
    lib.rtcSetGeometryMask(g, 0xFFFFFFFF)
    lib.rtcCommitGeometry(g)
    child = lib.rtcNewScene(dev)
    lib.rtcAttachGeometry(child, g)
    lib.rtcCommitScene(child)
    top = lib.rtcNewScene(dev)
    col = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 10], np.float32)
    lib.add_instance(dev, top, child, col)
    lib.rtcCommitScene(top)
    lib.check(dev)
    r = make_rayhits([[0, 0, 0]], [[0, 0, 1]])
    assert abs(lib.intersect(top, r.copy(), "1")["tfar"][0] - 9.0) < 1e-5
    vpad[:v.size] *= 2.0                                        # the child sphere grows to radius 2
    lib.rtcUpdateGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0)
    lib.rtcCommitGeometry(g)
    lib.rtcCommitScene(child)
    lib.rtcCommitScene(top)                                     # the instance geometry itself was not touched
    lib.check(dev)
    out = lib.intersect(top, r.copy(), "1")
    assert abs(out["tfar"][0] - 8.0) < 1e-5 and out["instID"][0] == 0, out
    lib.rtcReleaseGeometry(g)
    lib.rtcReleaseScene(child)
    lib.rtcReleaseScene(top)


def build_curve_scene(lib, dev, meshes, curves, quality=RTC_BUILD_QUALITY_MEDIUM):
    sc = lib.rtcNewScene(dev)
    lib.rtcSetSceneBuildQuality(sc, quality)
    keep = [lib.add_triangle_mesh(dev, sc, v, t, mask=mask, geom_id=gid)[1] for (v, t, gid, mask) in meshes]
    keep += [lib.add_round_linear_curves(dev, sc, c[0], c[1], c[2], mask=c[4], geom_id=c[3], flat=len(c) > 5 and c[5])[1] for c in curves]
    lib.rtcCommitScene(sc)
    lib.check(dev)
    return sc, keep


@pytest.mark.parametrize("name", ["curves", "curves_flat"])
@pytest.mark.parametrize("quality", [RTC_BUILD_QUALITY_LOW, RTC_BUILD_QUALITY_MEDIUM])
def test_curves_golden_all_entry_points(b200, quality, name):
    """RTC_GEOMETRY_TYPE_ROUND_LINEAR_CURVE (tutorials/hair_geometry's shipped model; roundline_intersector.h) and
    RTC_GEOMETRY_TYPE_FLAT_LINEAR_CURVE (line_intersector.h) against the reference's own outputs through every entry point:
    ids exact, t within 1e-4, u along the segment, v = 0, any-hit equal."""
    from tests.conftest import load_golden_curves
    lib, dev = b200
    g = load_golden_curves(name)
    sc, keep = build_curve_scene(lib, dev, g["meshes"], g["curves"], quality)
    b = RTCBounds()
    lib.rtcGetSceneBounds(sc, C.byref(b))
    got_b = np.array([b.lower_x, b.lower_y, b.lower_z, b.upper_x, b.upper_y, b.upper_z], np.float32)
    assert np.allclose(got_b, g["bounds"], rtol=1e-6, atol=1e-6) and (got_b[:3] <= g["bounds"][:3]).all() and (got_b[3:] >= g["bounds"][3:]).all()
    want = g["intersect_out"]
    for mode in MODES:
        got = lib.intersect(sc, g["rays_in"].copy(), mode)
        rep = compare_hits(want, got, TOL)
        assert rep["id_mismatch"] == 0 and rep["hit_miss_disagree"] == 0 and rep["tie"] <= 40, (mode, rep)   # ties: joints of two segments
        assert rep["max_rel_t"] <= TOL and rep["max_abs_uv"] <= TOL and rep["miss_untouched"], (mode, rep)
        ok = (got["geomID"] == want["geomID"]) & (got["primID"] == want["primID"]) & (got["geomID"] != 0xFFFFFFFF)
        for f in ("Ng_x", "Ng_y", "Ng_z"):
            assert np.allclose(got[f][ok], want[f][ok], rtol=1e-3, atol=1e-5), (mode, f)
        occ = lib.occluded(sc, rays_of(g["rays_in"]), mode)
        assert ((occ["tfar"] == -np.inf) == (g["occluded_out"]["tfar"] == -np.inf)).all(), mode
    lib.rtcReleaseScene(sc)


def test_curves_large_vs_oracle_and_errors(b200, oracle):
    """200 k curve segments + a triangle mesh against the C oracle, and the curve-specific error paths."""
    lib, dev = b200
    cv, ci, cf = scenes.hair_ball(25000, 8, seed=9, width=0.004)
    v, t = scenes.triangle_sphere(60)
    cv = cv.copy()
    cv[17, 0] = np.nan                       # invalid vertex: the segments that use it are dropped (scene_line_segments.h:427-441)
    cv[40, 3] = -1.0                         # negative radius: dropped as well
    sc, keep = build_curve_scene(lib, dev, [(v, t, 0, 0xFFFFFFFF)], [(cv, ci, cf, 1, 0xFFFFFFFF)])
    rng = np.random.RandomState(6)
    org = rng.normal(size=(300000, 3)).astype(np.float32)
    org = org / np.linalg.norm(org, axis=1, keepdims=True) * rng.uniform(1.02, 2.0, (300000, 1)).astype(np.float32)
    d = (-org + rng.normal(scale=0.7, size=org.shape)).astype(np.float32)
    rays = make_rayhits(org, d)
    got = lib.intersect(sc, rays.copy(), "1M")
    osc = oracle.scene([(v, t, 0, 0xFFFFFFFF)], curves=[(cv, ci, cf, 1, 0xFFFFFFFF)])
    want = osc.trace(rays.copy(), nthreads=16)
    from tests.parity import unexplained_curve_disagreements
    rep = compare_hits(want, got, TOL)
    assert (want["geomID"] == 1).sum() > 20000, rep
    # the only admissible differences are rays tangent to a segment (sign of the discriminant decided by rounding order)
    n_differ, unexplained = unexplained_curve_disagreements(rays, want, got, {1: (cv, ci)})
    assert n_differ <= 30 and unexplained == 0, (rep, n_differ, unexplained)
    assert rep["max_rel_t"] <= TOL and rep["max_abs_uv"] <= 2e-4, rep
    occ = lib.occluded(sc, rays_of(rays), "1M")
    wocc = osc.trace(rays_of(rays), occluded=True, nthreads=16)
    assert ((occ["tfar"] == -np.inf) != (wocc["tfar"] == -np.inf)).sum() <= n_differ
    osc.free()
    # an identity instance of the curve scene reports the same hits with instID set; curve buffers have their own formats
    top = lib.rtcNewScene(dev)
    lib.add_instance(dev, top, sc, np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], np.float32))
    lib.rtcCommitScene(top)
    lib.check(dev)
    sub = rays[:50000].copy()
    inst = lib.intersect(top, sub.copy(), "1M")
    hit = got["geomID"][:50000] != 0xFFFFFFFF
    assert (inst["instID"][hit] == 0).all() and (inst["instID"][~hit] == 0xFFFFFFFF).all()
    flat = inst.copy()
    flat["instID"] = got["instID"][:50000]            # everything but the instance id must agree with the un-instanced scene
    irep = compare_hits(got[:50000], flat, TOL)       # (the two segments that share a joint are hit at the same distance there and may swap: ties)
    assert irep["id_mismatch"] == 0 and irep["hit_miss_disagree"] == 0 and irep["tie"] <= 0.02 * irep["hits"] and irep["max_rel_t"] <= 1e-6, irep
    g = lib.rtcNewGeometry(dev, 16)
    lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, _ptr(cv), 0, 16, len(cv))
    assert lib.rtcGetDeviceError(dev) == 3                      # curves take FLOAT4 vertices
    lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT3, _ptr(ci), 0, 4, len(ci))
    assert lib.rtcGetDeviceError(dev) == 3                      # and one UINT per segment
    lib.rtcReleaseGeometry(g)
    lib.rtcReleaseScene(top)
    lib.rtcReleaseScene(sc)


def build_cubic_scene(lib, dev, meshes, cubics, quality=RTC_BUILD_QUALITY_MEDIUM):
    sc = lib.rtcNewScene(dev)
    lib.rtcSetSceneBuildQuality(sc, quality)
    keep = [lib.add_triangle_mesh(dev, sc, v, t, mask=mask, geom_id=gid)[1] for (v, t, gid, mask) in meshes]
    keep += [lib.add_flat_cubic_curves(dev, sc, c[0], c[1], c[4], c[5], c[6], mask=c[3], geom_id=c[2], round=len(c) > 7 and c[7])[1] for c in cubics]
    lib.rtcCommitScene(sc)
    lib.check(dev)
    return sc, keep


@pytest.mark.parametrize("name", ["curves_cubic", "curves_cubic_round"])
@pytest.mark.parametrize("quality", [RTC_BUILD_QUALITY_LOW, RTC_BUILD_QUALITY_MEDIUM])
def test_cubic_curves_golden_all_entry_points(b200, quality, name):
    """RTC_GEOMETRY_TYPE_FLAT_BEZIER / _BSPLINE / _CATMULL_ROM / _HERMITE_CURVE (curve_intersector_ribbon.h:73-190; tessellation
    rates default / 7 / 4 / 12, one geometry mask) and their ROUND counterparts (curve_intersector_sweep.h) against the
    reference's own outputs through every entry point: ids exact, t / u / v within tolerance, Ng = the curve tangent (flat) or
    the surface normal (round), any-hit equal, scene bounds as the reference reports them."""
    from tests.conftest import load_golden_cubic
    lib, dev = b200
    g = load_golden_cubic(name)
    sc, keep = build_cubic_scene(lib, dev, g["meshes"], g["cubics"], quality)
    b = RTCBounds()
    lib.rtcGetSceneBounds(sc, C.byref(b))
    got_b = np.array([b.lower_x, b.lower_y, b.lower_z, b.upper_x, b.upper_y, b.upper_z], np.float32)
    assert np.allclose(got_b, g["bounds"], rtol=1e-6, atol=1e-6) and (got_b[:3] <= g["bounds"][:3]).all() and (got_b[3:] >= g["bounds"][3:]).all()
    want = g["intersect_out"]
    for mode in MODES:
        got = lib.intersect(sc, g["rays_in"].copy(), mode)
        rep = compare_hits(want, got, TOL)
        assert rep["id_mismatch"] == 0 and rep["hit_miss_disagree"] == 0 and rep["tie"] <= 4, (mode, rep)
        # u of a round curve is the root of a Newton iteration: ill-conditioned where the ray grazes the tube (seen: 2.5e-3)
        assert rep["max_rel_t"] <= TOL and rep["max_abs_uv"] <= (5e-3 if name.endswith("round") else 2e-4) and rep["miss_untouched"], (mode, rep)
        ok = (got["geomID"] == want["geomID"]) & (got["primID"] == want["primID"]) & (got["geomID"] != 0xFFFFFFFF)
        for f in ("Ng_x", "Ng_y", "Ng_z"):
            assert np.allclose(got[f][ok], want[f][ok], rtol=2e-2 if name.endswith("round") else 1e-3, atol=1e-4 if name.endswith("round") else 1e-5), (mode, f)
        occ = lib.occluded(sc, rays_of(g["rays_in"]), mode)
        assert ((occ["tfar"] == -np.inf) == (g["occluded_out"]["tfar"] == -np.inf)).all(), mode
    lib.rtcReleaseScene(sc)


@pytest.mark.parametrize("basis", ["bezier", "bspline", "catmull_rom", "hermite"])
def test_round_cubic_curves_large_vs_oracle(b200, oracle, basis):
    """20 000 strands of ROUND cubic curves + a triangle mesh against the C oracle.  The device runs the oracle's arithmetic
    operation for operation (tests/test_emu_core.py), but the BVH holds the 7 first-level sub-segments of a curve as separate
    primitives, so candidates shorten the ray in another order than in the oracle's whole-curve loop -- and the iteration's start
    value for an exit point depends on the current tfar (curve_intersector_sweep.h:216-217).  Hence: nearly all hits bit-identical,
    the rest explained as silhouette grazes, no more of them than the reference has between its own ISA paths."""
    from tests.parity import sweep_disagreements
    lib, dev = b200
    cv, ci, tg = scenes.cubic_hair(20000, basis, seed=12, width=0.006)
    v, t = scenes.triangle_sphere(60)
    sc, keep = build_cubic_scene(lib, dev, [(v, t, 0, 0xFFFFFFFF)], [(cv, ci, 1, 0xFFFFFFFF, basis, None, tg, True)])
    rng = np.random.RandomState(8)
    org = rng.normal(size=(200000, 3)).astype(np.float32)
    org = org / np.linalg.norm(org, axis=1, keepdims=True) * rng.uniform(1.02, 2.0, (200000, 1)).astype(np.float32)
    d = (-org + rng.normal(scale=0.7, size=org.shape)).astype(np.float32)
    rays = make_rayhits(org, d)
    got = lib.intersect(sc, rays.copy(), "1M")
    osc = oracle.scene([(v, t, 0, 0xFFFFFFFF)], cubics=[(cv, ci, 1, 0xFFFFFFFF, basis, 4, tg, True)])
    want = osc.trace(rays.copy(), nthreads=16)
    assert (want["geomID"] == 1).sum() > 15000
    n_differ, unexplained = sweep_disagreements(rays, want, got, {1})
    assert n_differ <= 40 and unexplained <= 4, (n_differ, unexplained)          # 2e-4 / 2e-5 of the rays
    same = (got["geomID"] == want["geomID"]) & (got["primID"] == want["primID"]) & (want["geomID"] == 1)
    exact = np.ones(len(rays), bool)
    for f in ("tfar", "u", "v", "Ng_x", "Ng_y", "Ng_z"):
        exact &= got[f].view(np.uint32) == want[f].view(np.uint32)
    assert (exact & same).sum() >= 0.998 * same.sum(), ((exact & same).sum(), same.sum())
    tri = want["geomID"] == 0                                                      # triangle hits are untouched by all this
    assert (got["primID"][tri & (got["geomID"] == 0)] == want["primID"][tri & (got["geomID"] == 0)]).all()
    occ = lib.occluded(sc, rays_of(rays), "1M")
    wocc = osc.trace(rays_of(rays), occluded=True, nthreads=16)
    assert ((occ["tfar"] == -np.inf) != (wocc["tfar"] == -np.inf)).sum() <= n_differ
    osc.free()
    lib.rtcReleaseScene(sc)


@pytest.mark.parametrize("basis,tess", [("bezier", None), ("bspline", 9), ("catmull_rom", 16), ("hermite", 1)])
def test_cubic_curves_large_vs_oracle(b200, oracle, basis, tess):
    """30 000 strands of cubic curves + a triangle mesh against the C oracle.  The device runs the oracle's arithmetic operation
    for operation (tests/test_emu_core.py), so the hits must be bit-identical wherever the two name the same curve, the GPU
    may lose no hit (conservative curve bounds in the BVH), and a different curve is only admissible at the same distance."""
    lib, dev = b200
    cv, ci, tg = scenes.cubic_hair(30000, basis, seed=11, width=0.004)
    cv = cv.copy()
    cv[25, 1] = np.inf                          # an invalid control point drops the curves that use it (scene_curves.h:498-533)
    v, t = scenes.triangle_sphere(60)
    sc, keep = build_cubic_scene(lib, dev, [(v, t, 0, 0xFFFFFFFF)], [(cv, ci, 1, 0xFFFFFFFF, basis, tess, tg)])
    rng = np.random.RandomState(6)
    org = rng.normal(size=(300000, 3)).astype(np.float32)
    org = org / np.linalg.norm(org, axis=1, keepdims=True) * rng.uniform(1.02, 2.0, (300000, 1)).astype(np.float32)
    d = (-org + rng.normal(scale=0.7, size=org.shape)).astype(np.float32)
    rays = make_rayhits(org, d)
    got = lib.intersect(sc, rays.copy(), "1M")
    osc = oracle.scene([(v, t, 0, 0xFFFFFFFF)], cubics=[(cv, ci, 1, 0xFFFFFFFF, basis, 4 if tess is None else tess, tg)])
    want = osc.trace(rays.copy(), nthreads=16)
    rep = compare_hits(want, got, TOL)
    assert (want["geomID"] == 1).sum() > 20000, rep
    assert rep["hit_miss_disagree"] == 0 and rep["id_mismatch"] == 0 and rep["tie"] <= 20, rep
    same = (got["geomID"] == want["geomID"]) & (got["primID"] == want["primID"]) & (want["geomID"] == 1)
    for f in ("tfar", "u", "v", "Ng_x", "Ng_y", "Ng_z"):
        assert (got[f][same].view(np.uint32) == want[f][same].view(np.uint32)).all(), f
    occ = lib.occluded(sc, rays_of(rays), "1M")
    wocc = osc.trace(rays_of(rays), occluded=True, nthreads=16)
    assert ((occ["tfar"] == -np.inf) == (wocc["tfar"] == -np.inf)).all()
    osc.free()
    lib.rtcReleaseScene(sc)


def test_cubic_curve_api_errors(b200):
    """Curve-specific API behaviour: the tessellation rate exists for cubic curves only and is clamped to 1..16
    (scene_curves.cpp:244-249), a Hermite geometry needs its tangent buffer, formats are FLOAT4 / UINT."""
    lib, dev = b200
    cv, ci, tg = scenes.cubic_hair(300, "hermite", seed=3, width=0.05)
    g = lib.rtcNewGeometry(dev, 0)
    lib.rtcSetGeometryTessellationRate(g, 8.0)
    assert lib.rtcGetDeviceError(dev) == 3                      # triangle mesh: operation not supported
    lib.rtcReleaseGeometry(g)
    g = lib.rtcNewGeometry(dev, 25)                             # flat Bezier: no tangent buffer
    lib.rtcSetSharedGeometryBuffer(g, 4, 0, 0x9004, _ptr(tg), 0, 16, len(tg))
    assert lib.rtcGetDeviceError(dev) == 2
    lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, _ptr(cv), 0, 16, len(cv))
    assert lib.rtcGetDeviceError(dev) == 3
    lib.rtcReleaseGeometry(g)
    sc = lib.rtcNewScene(dev)
    g = lib.rtcNewGeometry(dev, 41)                             # flat Hermite without tangents: the commit fails
    lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0, 0x9004, _ptr(cv), 0, 16, len(cv))
    lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_INDEX, 0, 0x5001, _ptr(ci), 0, 4, len(ci))
    lib.rtcSetGeometryTessellationRate(g, 100.0)                # clamped to 16
    lib.rtcCommitGeometry(g)
    lib.rtcAttachGeometry(sc, g)
    lib.rtcCommitScene(sc)
    assert lib.rtcGetDeviceError(dev) == 3
    lib.rtcSetSharedGeometryBuffer(g, 4, 0, 0x9004, _ptr(tg), 0, 16, len(tg))
    lib.rtcCommitGeometry(g)
    lib.rtcCommitScene(sc)
    lib.check(dev)
    rays = make_rayhits(np.array([[0, 0, 3]], np.float32).repeat(64, 0) + np.random.RandomState(1).normal(scale=0.2, size=(64, 3)).astype(np.float32),
                        np.tile([[0, 0, -1]], (64, 1)))
    out = lib.intersect(sc, rays.copy(), "1M")
    hit = out["geomID"] != 0xFFFFFFFF
    assert hit.any() and (np.abs(out["v"][hit]) <= 1.0 + 1e-5).all() and ((out["u"][hit] >= 0) & (out["u"][hit] <= 1)).all()
    lib.rtcReleaseGeometry(g)
    lib.rtcReleaseScene(sc)


def test_interpolate_matches_the_reference(b200):
    """rtcInterpolate on triangle and quad meshes (scene_triangle_mesh.h:49-105, scene_quad_mesh.h): P, dPdu, dPdv of the vertex
    buffer at (primID, u, v) -- what shading code calls with the u, v of a hit -- bit-equal to the reference's at the reference's
    own hits of the golden fixture, and equal to the hit point org + t dir of a traced ray."""
    from embree_b200.rtc import InterpolateArguments
    lib, dev = b200
    meshes, rin, want_i, _o, _b = load_golden("quads")
    sc, keep = build_scene(lib, dev, meshes)
    got = lib.intersect(sc, rin.copy(), "1M")

    def interp(L, scn, gid, prim, u, v):
        P, du, dv = (C.c_float * 3)(), (C.c_float * 3)(), (C.c_float * 3)()
        a = InterpolateArguments(L.rtcGetGeometry(scn, gid), prim, u, v, RTC_BUFFER_TYPE_VERTEX, 0, C.cast(P, C.c_void_p), C.cast(du, C.c_void_p),
                                 C.cast(dv, C.c_void_p), None, None, None, 3)
        L.rtcInterpolate(C.byref(a))
        return np.array([list(P), list(du), list(dv)], np.float32)
    hits = np.nonzero(got["geomID"] != 0xFFFFFFFF)[0][:400]
    assert len(hits) > 200 and len(set(got["geomID"][hits])) >= 2          # quad meshes and the triangle mesh
    for i in hits:
        r = got[i]
        mine = interp(lib, sc, int(r["geomID"]), int(r["primID"]), float(r["u"]), float(r["v"]))
        hitp = np.array([r["org_x"] + r["tfar"] * r["dir_x"], r["org_y"] + r["tfar"] * r["dir_y"], r["org_z"] + r["tfar"] * r["dir_z"]], np.float64)
        assert np.abs(mine[0] - hitp).max() <= 2e-5 * max(1.0, np.abs(hitp).max()), (i, mine[0], hitp)
    queries = want_i[np.nonzero(want_i["geomID"] != 0xFFFFFFFF)[0][:400]]

    def run(R):
        rdev = R.new_device(None)
        rsc, rkeep = build_scene(R, rdev, meshes)
        out = np.stack([interp(R, rsc, int(q["geomID"]), int(q["primID"]), float(q["u"]), float(q["v"])) for q in queries])
        R.rtcReleaseScene(rsc)
        R.rtcReleaseDevice(rdev)
        return {"interp": out}
    ref = reference_outputs("interpolate_quads", run)[0]["interp"]
    assert len(ref) == len(queries) > 200
    for j, q in enumerate(queries):
        mine = interp(lib, sc, int(q["geomID"]), int(q["primID"]), float(q["u"]), float(q["v"]))
        assert (ref[j].view(np.uint32) == mine.view(np.uint32)).all(), j
    lib.check(dev)
    lib.rtcReleaseScene(sc)


def test_update_and_recommit(b200):
    """UpdateTest (verify.cpp:1835) / dynamic_scene: move the vertices, rtcUpdateGeometryBuffer, re-commit."""
    lib, dev = b200
    v, t = scenes.triangle_sphere(10)
    v = v.copy()
    vpad = np.zeros(v.size + 4, np.float32)
    vpad[:v.size] = v.ravel()
    g = lib.rtcNewGeometry(dev, RTC_GEOMETRY_TYPE_TRIANGLE)
    lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, _ptr(vpad), 0, 12, len(v))
    lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT3, _ptr(t), 0, 12, len(t))
    lib.rtcSetGeometryMask(g, 0xFFFFFFFF)
    lib.rtcCommitGeometry(g)
    sc = lib.rtcNewScene(dev)
    lib.rtcSetSceneFlags(sc, 1)  # DYNAMIC
    lib.rtcSetSceneBuildQuality(sc, RTC_BUILD_QUALITY_LOW)
    lib.rtcAttachGeometry(sc, g)
    lib.rtcCommitScene(sc)
    r = make_rayhits([[0, 0, -5]], [[0, 0, 1]])
    assert abs(lib.intersect(sc, r.copy(), "1")["tfar"][0] - 4.0) < 1e-5
    vpad[:v.size] *= 2.0
    lib.rtcUpdateGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0)
    lib.rtcCommitGeometry(g)
    lib.rtcCommitScene(sc)
    assert abs(lib.intersect(sc, r.copy(), "1")["tfar"][0] - 3.0) < 1e-5
    lib.check(dev)
    lib.rtcReleaseGeometry(g)
    lib.rtcReleaseScene(sc)


@pytest.mark.parametrize("scene_quality", [RTC_BUILD_QUALITY_LOW, RTC_BUILD_QUALITY_MEDIUM])
def test_refit_matches_rebuild(b200, oracle, scene_quality):
    """RTC_BUILD_QUALITY_REFIT on the geometry (kernels/bvh/bvh_refit.cpp; verify.cpp update.* benchmarks): the first commit
    builds, later commits with moved vertices and unchanged topology refit the same BVH8 (builder == 2).  Hits after a
    refit equal the oracle's on the moved mesh and a from-scratch rebuild's; a primitive-count change falls back to a build."""
    lib, dev = b200
    v, t = scenes.triangle_sphere(80)
    sc = lib.rtcNewScene(dev)
    lib.rtcSetSceneFlags(sc, 1)            # DYNAMIC
    lib.rtcSetSceneBuildQuality(sc, scene_quality)
    g = lib.rtcNewGeometry(dev, RTC_GEOMETRY_TYPE_TRIANGLE)
    vpad = np.zeros(v.size + 4, np.float32)
    vpad[:v.size] = v.ravel()
    lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, _ptr(vpad), 0, 12, len(v))
    lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT3, _ptr(t), 0, 12, len(t))
    lib.rtcSetGeometryMask(g, 0xFFFFFFFF)
    lib.rtcSetGeometryBuildQuality(g, 3)   # RTC_BUILD_QUALITY_REFIT
    lib.rtcCommitGeometry(g)
    lib.rtcAttachGeometry(sc, g)
    lib.rtcCommitScene(sc)
    lib.check(dev)
    assert lib.scene_stats(sc).builder in (0, 1)
    rng = np.random.RandomState(4)
    rays = scenes.as_numpy_rayhits(scenes.incoherent_rays_reference(100000, org=(0.1, -0.2, 0.05)))
    for frame in range(3):
        v2 = (v * np.array([1.0 + 0.3 * frame, 1.0, 1.0 - 0.2 * frame], np.float32) + rng.normal(scale=2e-3, size=v.shape)).astype(np.float32)
        vpad[:v.size] = v2.ravel()
        lib.rtcUpdateGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0)
        lib.rtcCommitGeometry(g)
        lib.rtcCommitScene(sc)
        lib.check(dev)
        assert lib.scene_stats(sc).builder == 2, "expected a refit"
        b = RTCBounds()
        lib.rtcGetSceneBounds(sc, C.byref(b))
        used = v2[t.ravel()]                 # bounds cover the vertices triangles reference (the generator leaves spare pole copies)
        assert np.array_equal(np.array([b.lower_x, b.lower_y, b.lower_z, b.upper_x, b.upper_y, b.upper_z], np.float32), np.concatenate([used.min(0), used.max(0)]))
        got = lib.intersect(sc, rays.copy(), "1M")
        want = oracle.trace(v2, t, rays.copy(), nthreads=8)
        rep = compare_hits(want, got, TOL, meshes=[(v2, t, 0, 0xFFFFFFFF)])
        assert rep["id_mismatch"] == 0 and rep["hit_miss_disagree"] == 0 and rep["max_rel_t"] <= TOL and rep["ng_bit_exact"], (frame, rep)
        fresh, keep = build_scene(lib, dev, [(v2, t, 0, 0xFFFFFFFF)], scene_quality)
        got2 = lib.intersect(fresh, rays.copy(), "1M")
        rep2 = compare_hits(got2, got, TOL, meshes=[(v2, t, 0, 0xFFFFFFFF)])
        assert rep2["id_mismatch"] == 0 and rep2["hit_miss_disagree"] == 0 and rep2["max_rel_t"] == 0.0, (frame, rep2)
        occ = lib.occluded(sc, rays_of(rays), "1M")
        assert ((occ["tfar"] == -np.inf) == (got["geomID"] != 0xFFFFFFFF)).all()
        lib.rtcReleaseScene(fresh)
    # a vertex turning NaN invalidates its triangles (scene_triangle_mesh.h:194-215) -- also under refit
    vpad[0:3] = np.nan
    lib.rtcUpdateGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0)
    lib.rtcCommitGeometry(g)
    lib.rtcCommitScene(sc)
    lib.check(dev)
    got = lib.intersect(sc, rays.copy(), "1M")
    v3 = vpad[:v.size].reshape(-1, 3).copy()
    want = oracle.trace(v3, t, rays.copy(), nthreads=8)
    rep = compare_hits(want, got, TOL)
    assert rep["id_mismatch"] == 0 and rep["hit_miss_disagree"] == 0, rep
    lib.rtcReleaseGeometry(g)
    lib.rtcReleaseScene(sc)


@pytest.mark.parametrize("quality", [RTC_BUILD_QUALITY_LOW, RTC_BUILD_QUALITY_MEDIUM])
def test_watertight_and_reference_side_by_side(b200, oracle, quality):
    """WatertightTest (verify.cpp:3611-3690, <= 2e-5 leaks) + 200k-ray parity against the oracle and the unmodified reference
    (traced on the host cores when oracle/_ref is built, else its stored answers for every 50th ray)."""
    lib, dev = b200
    v, t = scenes.triangle_sphere(201)
    sc, keep = build_scene(lib, dev, [(v, t, 0, 0xFFFFFFFF)], quality)
    rays = scenes.as_numpy_rayhits(scenes.incoherent_rays_reference(200000, org=(0.05, -0.1, 0.02)))
    got = lib.intersect(sc, rays.copy(), "1M")
    assert (got["geomID"] == 0xFFFFFFFF).mean() <= 2e-5
    want = oracle.trace(v, t, rays.copy(), nthreads=8)
    rep = assert_parity(want, got, allow_ties=2)
    assert rep["ng_bit_exact"]

    def run(R):
        from tests.parity import api_trace_mt
        rd = R.new_device(None)
        rs = R.rtcNewScene(rd)
        _, k2 = R.add_triangle_mesh(rd, rs, v, t, mask=0xFFFFFFFF)
        R.rtcCommitScene(rs)
        ref = api_trace_mt(R, rs, rays.copy(), 16)
        R.rtcReleaseScene(rs)
        R.rtcReleaseDevice(rd)
        return {"hits": ref}
    out, rows = reference_outputs("watertight_sphere201", run, {"hits": rays}, stride=50)   # the reference's scene does not depend on `quality`
    ref, got = out["hits"], got[rows]
    # the reference's fast path itself leaks ~1e-6 of edge rays (SURVEY 7.4): those are not parity failures
    both = (ref["geomID"] != 0xFFFFFFFF)
    rep = compare_hits(ref[both], got[both], TOL)
    assert rep["id_mismatch"] == 0 and rep["tie"] <= 2 and rep["max_rel_t"] <= TOL and rep["max_abs_uv"] <= TOL, rep
    assert (~both).mean() <= 2e-5
    lib.rtcReleaseScene(sc)


def test_robust_watertight_and_reference(b200, oracle):
    """RTC_SCENE_FLAG_ROBUST at scale: no leaks at all from inside a closed 160 k-triangle sphere, ids equal to the
    oracle's Pluecker path for 400 k rays and to the reference's (live when oracle/_ref is built, else its stored answers for
    every 100th ray)."""
    lib, dev = b200
    v, t = scenes.triangle_sphere(201)
    sc, keep = build_scene(lib, dev, [(v, t, 0, 0xFFFFFFFF)], RTC_BUILD_QUALITY_MEDIUM, flags=4)
    rays = scenes.as_numpy_rayhits(scenes.incoherent_rays_reference(400000, org=(0.05, -0.1, 0.02)))
    got = lib.intersect(sc, rays.copy(), "1M")
    assert (got["geomID"] == 0).all()
    want = oracle.scene([(v, t, 0, 0xFFFFFFFF)], robust=True).trace(rays.copy(), nthreads=8)
    rep = assert_parity(want, got, allow_ties=4)
    assert rep["ng_bit_exact"]
    occ = lib.occluded(sc, rays_of(rays), "1M")
    assert (occ["tfar"] == -np.inf).all()

    def run(R):
        from tests.parity import api_trace_mt
        rd = R.new_device(None)
        rs = R.rtcNewScene(rd)
        R.rtcSetSceneFlags(rs, 4)
        _, k2 = R.add_triangle_mesh(rd, rs, v, t, mask=0xFFFFFFFF)
        R.rtcCommitScene(rs)
        ref = api_trace_mt(R, rs, rays.copy(), 16)
        R.rtcReleaseScene(rs)
        R.rtcReleaseDevice(rd)
        return {"hits": ref}
    out, rows = reference_outputs("robust_sphere201", run, {"hits": rays}, stride=100)
    assert_parity(out["hits"], got[rows], allow_ties=4)
    lib.rtcReleaseScene(sc)


def test_full_size_properties_1m(b200, oracle):
    """BASELINE config sizes (1 002 000-triangle sphere, 4 Mi rays) through size-independent properties:
    rays from inside the closed sphere hit (leaks <= 2e-5 as WatertightTest allows -- the per-triangle edge tests of
    Moeller-Trumbore are not watertight in the reference either -- and every leaked ray is one the oracle leaks too);
    hit points lie on the sphere; occluded == (intersect found a hit); re-tracing with tfar = t*(1+eps) returns the
    same primitive (idempotence); LOW and MEDIUM builders agree on every id."""
    import torch
    lib, dev = b200
    v, t = scenes.triangle_sphere(501)
    n = 1 << 22
    rays_t = scenes.incoherent_rays_reference(n)
    rays = scenes.as_numpy_rayhits(rays_t)
    results = []
    for quality in (RTC_BUILD_QUALITY_LOW, RTC_BUILD_QUALITY_MEDIUM):
        sc, keep = build_scene(lib, dev, [(v, t, 0, 0xFFFFFFFF)], quality)
        assert lib.scene_stats(sc).num_triangles == 1002000
        got = lib.intersect(sc, rays.copy(), "1M")
        hit = got["geomID"] == 0
        assert (~hit).mean() <= 2e-5 and (got["geomID"][~hit] == 0xFFFFFFFF).all()
        if (~hit).any():
            chk = oracle.trace(v, t, rays[~hit].copy())
            assert (chk["geomID"] == 0xFFFFFFFF).all()       # the same rays leak through the reference algorithm
        P = np.stack([got[f"dir_{a}"][hit] * got["tfar"][hit] for a in "xyz"], 1)
        rad = np.linalg.norm(P, axis=1)
        assert rad.min() > 0.9999 and rad.max() < 1.00001
        occ = lib.occluded(sc, rays_of(rays), "1M")
        assert ((occ["tfar"] == -np.inf) == hit).all()
        again = rays.copy()
        again["tfar"] = np.where(hit, got["tfar"] * np.float32(1.000001), np.float32(np.inf))
        again = lib.intersect(sc, again, "16M")
        assert (again["primID"] == got["primID"]).all()
        results.append(got)
        lib.rtcReleaseScene(sc)
    rep = compare_hits(results[0], results[1], TOL)
    assert rep["id_mismatch"] == 0 and rep["tie"] <= 8 and rep["max_rel_t"] <= TOL, rep


def _dynamic_meshes(n, seed=4):
    """n triangle spheres of different sizes scattered in a box, as tutorials/dynamic_scene places its spheres."""
    rng = np.random.RandomState(seed)
    out = []
    for i in range(n):
        v, t = scenes.triangle_sphere(int(rng.randint(6, 24)))
        c = rng.uniform(-3, 3, 3).astype(np.float32)
        r = np.float32(rng.uniform(0.2, 0.9))
        out.append(((v * r + c).astype(np.float32), t.copy()))
    return out


@pytest.mark.parametrize("robust", [False, True])
@pytest.mark.parametrize("scene_quality", [RTC_BUILD_QUALITY_LOW, RTC_BUILD_QUALITY_MEDIUM])
def test_two_level_dynamic_scene(b200, oracle, scene_quality, robust):
    """a25: an RTC_SCENE_FLAG_DYNAMIC scene of several triangle meshes keeps one BVH per mesh (bvh_builder_twolevel.cpp:35-240) when only
    some of them were modified since the last commit: the commit rebuilds / refits only those (scene.cpp:878-884) and re-assembles the
    top level; when (nearly) everything moved, one rebuild over all triangles is cheaper and is what happens.  Hits equal the oracle's
    single BVH over the same triangles at every stage: first commit, one mesh moved (kept BVHs are built), another one moved, all moved,
    one mesh refitted, a mesh disabled, a mesh with a new triangle count (new layout), a slot changing hands, a single mesh left."""
    lib, dev = b200
    meshes = _dynamic_meshes(24)
    sc = lib.rtcNewScene(dev)
    lib.rtcSetSceneFlags(sc, 1 | (4 if robust else 0))   # DYNAMIC (| ROBUST)
    lib.rtcSetSceneBuildQuality(sc, scene_quality)
    geoms, bufs = [], []
    for i, (v, t) in enumerate(meshes):
        vpad = np.zeros(v.size + 4, np.float32)
        vpad[:v.size] = v.ravel()
        g = lib.rtcNewGeometry(dev, RTC_GEOMETRY_TYPE_TRIANGLE)
        lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, _ptr(vpad), 0, 12, len(v))
        lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT3, _ptr(t), 0, 12, len(t))
        lib.rtcSetGeometryMask(g, 0xFFFFFFFF)
        if i == 5:
            lib.rtcSetGeometryBuildQuality(g, 3)          # RTC_BUILD_QUALITY_REFIT for this one
        lib.rtcCommitGeometry(g)
        lib.rtcAttachGeometryByID(sc, g, i)
        geoms.append(g)
        bufs.append((vpad, v.shape[0], t))
    rng = np.random.RandomState(9)
    org = rng.uniform(-5, 5, (40000, 3)).astype(np.float32)
    d = rng.normal(size=(40000, 3)).astype(np.float32)
    rays = make_rayhits(org, d)
    enabled = [True] * len(meshes)

    def check(stage):
        lib.rtcCommitScene(sc)
        lib.check(dev)
        cur = [(bufs[i][0][:bufs[i][1] * 3].reshape(-1, 3).copy(), bufs[i][2], i, 0xFFFFFFFF) for i in range(len(bufs)) if enabled[i]]
        want = oracle.scene(cur, robust=robust).trace(rays.copy(), nthreads=8)
        got = lib.intersect(sc, rays.copy(), "1M")
        rep = compare_hits(want, got, TOL, meshes=cur)
        assert rep["id_mismatch"] == 0 and rep["hit_miss_disagree"] == 0 and rep["tie"] <= 12, (stage, rep)
        assert rep["max_rel_t"] <= TOL and rep["hits"] > (2500 if sum(enabled) > 1 else 30), (stage, rep)
        occ = lib.occluded(sc, rays_of(rays), "1M")
        assert ((occ["tfar"] == -np.inf) == (want["geomID"] != 0xFFFFFFFF)).all(), stage
        return lib.scene_stats(sc)
    st = check("first commit")
    assert st.builder != 3 and st.num_triangles == sum(len(t) for (_v, t) in meshes)   # everything is new: one BVH over all of it is cheaper
    # one mesh moves: the two-level path takes over (and builds the kept BVH of every mesh, once)
    bufs[2][0][:bufs[2][1] * 3] += np.float32(0.35)
    lib.rtcUpdateGeometryBuffer(geoms[2], RTC_BUFFER_TYPE_VERTEX, 0)
    lib.rtcCommitGeometry(geoms[2])
    l0 = lib.rtcb200GetLaunchCount()
    st = check("one mesh moved")
    all_launches = lib.rtcb200GetLaunchCount() - l0
    assert st.builder == 3
    # another mesh moves: only that mesh is rebuilt (far fewer kernel launches than when all 24 kept BVHs were built)
    bufs[3][0][:bufs[3][1] * 3] -= np.float32(0.25)
    lib.rtcUpdateGeometryBuffer(geoms[3], RTC_BUFFER_TYPE_VERTEX, 0)
    lib.rtcCommitGeometry(geoms[3])
    l0 = lib.rtcb200GetLaunchCount()
    st = check("another mesh moved")
    assert st.builder == 3 and lib.rtcb200GetLaunchCount() - l0 < all_launches / 5 + 40   # (the traces of check() are part of both counts)
    # every mesh moves in one frame (tutorials/dynamic_scene): one rebuild over everything is cheaper again; then back
    for i in range(len(geoms)):
        bufs[i][0][:bufs[i][1] * 3] += np.float32(0.01)
        lib.rtcUpdateGeometryBuffer(geoms[i], RTC_BUFFER_TYPE_VERTEX, 0)
        lib.rtcCommitGeometry(geoms[i])
    assert check("all meshes moved").builder != 3
    bufs[4][0][:bufs[4][1] * 3] += np.float32(0.15)
    lib.rtcUpdateGeometryBuffer(geoms[4], RTC_BUFFER_TYPE_VERTEX, 0)
    lib.rtcCommitGeometry(geoms[4])
    assert check("one mesh moved again").builder == 3
    # the REFIT mesh deforms
    bufs[5][0][:bufs[5][1] * 3] *= np.float32(1.1)
    lib.rtcUpdateGeometryBuffer(geoms[5], RTC_BUFFER_TYPE_VERTEX, 0)
    lib.rtcCommitGeometry(geoms[5])
    check("refit mesh deformed")
    # a mesh is disabled, another one gets a different triangle count (fewer triangles through a shorter index buffer)
    lib.rtcDisableGeometry(geoms[7])
    enabled[7] = False
    t9 = bufs[9][2][: len(bufs[9][2]) // 2].copy()
    lib.rtcSetSharedGeometryBuffer(geoms[9], RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT3, _ptr(t9), 0, 12, len(t9))
    lib.rtcCommitGeometry(geoms[9])
    bufs[9] = (bufs[9][0], bufs[9][1], t9)
    check("disabled + new triangle count")
    # a slot changes hands between two meshes of identical size in ONE commit (same node / record counts: the layout is reused)
    vtw, ttw = scenes.triangle_sphere(12)
    for i, c in ((20, (-2.0, 2.0, 1.0)), (21, (2.5, -1.0, -2.0))):
        vv = (vtw * np.float32(0.5) + np.float32(c)).astype(np.float32)
        vpad = np.zeros(vv.size + 4, np.float32)
        vpad[:vv.size] = vv.ravel()
        tcp = ttw.copy()
        lib.rtcSetSharedGeometryBuffer(geoms[i], RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, _ptr(vpad), 0, 12, len(vv))
        lib.rtcSetSharedGeometryBuffer(geoms[i], RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT3, _ptr(tcp), 0, 12, len(tcp))
        lib.rtcCommitGeometry(geoms[i])
        bufs[i] = (vpad, len(vv), tcp)
    lib.rtcDisableGeometry(geoms[21])
    enabled[21] = False
    check("two equal meshes, one disabled")
    lib.rtcDisableGeometry(geoms[20])
    lib.rtcEnableGeometry(geoms[21])
    enabled[20], enabled[21] = False, True
    check("slot handed to the other equal mesh")
    # a mesh is REPLACED by a new geometry object of the same size, set up by the same sequence of calls (same modification counter)
    # and very likely allocated where the released one lived: the kept BVH of the old object must not be taken for the new one's
    v11 = (bufs[11][0][:bufs[11][1] * 3].reshape(-1, 3) + np.float32(0.6)).astype(np.float32)
    lib.rtcDetachGeometry(sc, 11)
    lib.rtcReleaseGeometry(geoms[11])
    vpad = np.zeros(v11.size + 4, np.float32)
    vpad[:v11.size] = v11.ravel()
    g = lib.rtcNewGeometry(dev, RTC_GEOMETRY_TYPE_TRIANGLE)
    lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, _ptr(vpad), 0, 12, len(v11))
    lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT3, _ptr(bufs[11][2]), 0, 12, len(bufs[11][2]))
    lib.rtcSetGeometryMask(g, 0xFFFFFFFF)
    lib.rtcCommitGeometry(g)
    lib.rtcAttachGeometryByID(sc, g, 11)
    geoms[11] = g
    bufs[11] = (vpad, len(v11), bufs[11][2])
    assert check("mesh replaced by a new geometry object").builder == 3
    # leaving the two-level regime: all but one mesh disabled -> the ordinary single BVH
    for i in range(1, len(geoms)):
        if enabled[i]:
            lib.rtcDisableGeometry(geoms[i])
            enabled[i] = False
    st = check("single mesh left")
    assert st.builder != 3
    for g in geoms:
        lib.rtcReleaseGeometry(g)
    lib.rtcReleaseScene(sc)
