"""Instance traversal: scenes with instances committed with one BVH per instanced scene and a top level over the scene's own
primitives and one primitive per instance, instead of flattened copies.  rtcb200SetTuning("instance_flatten_max", 0) forces the
path on every scene with instances; each test holds it to the reference's stored answers, to the C oracle, or byte for byte to the
flattened path on the same rays (ties at bit-identical t excepted: the traversal order decides which of two such records wins)."""
import ctypes as C
import re

import numpy as np
import pytest

from embree_b200 import scenes
import embree_b200
from embree_b200.rtc import (RAYHIT_DTYPE, RTC_BUFFER_TYPE_VERTEX, RTC_BUILD_QUALITY_LOW, RTC_BUILD_QUALITY_MEDIUM,
                             RTC_FORMAT_FLOAT3X4_COLUMN_MAJOR, RTCBounds, _ptr, make_rayhits, rays_of)
from tests.conftest import load_golden_instances
from tests.parity import build_instanced_hair, compare_hits, explain_hit_miss, instanced_hair_scene
from tests.test_gpu_parity import MODES, TOL, assert_parity, build_instanced, build_scene
from tests.test_trace_schedules import SHIPPED, _cuda, _stream, ray_mix, tuning

NO_HIT = 0xFFFFFFFF


def test_flatten_max_is_a_tuning_key():
    """The selection threshold is settable like every other key and refuses a negative value."""
    lib = embree_b200.load()
    assert "instance_flatten_max" in SHIPPED and SHIPPED["instance_flatten_max"] > 0
    assert lib.rtcb200SetTuning(b"instance_flatten_max", -1) == -1
    with tuning(lib, instance_flatten_max=0):
        pass


def traversal(lib, fn, *a, **k):
    """fn(*a, **k) with every commit in it taking instance traversal"""
    with tuning(lib, instance_flatten_max=0):
        return fn(*a, **k)


def bounds(lib, sc):
    b = RTCBounds()
    lib.rtcGetSceneBounds(sc, C.byref(b))
    return np.array([b.lower_x, b.lower_y, b.lower_z, b.upper_x, b.upper_y, b.upper_z], np.float32)


def same_but_ties(got, want, what, max_ties):
    """Records byte-identical, except rays whose two answers are hits at the same t (bit for bit) on different records."""
    g = np.ascontiguousarray(got).view(np.uint8).reshape(len(got), -1)
    w = np.ascontiguousarray(want).view(np.uint8).reshape(len(want), -1)
    bad = np.nonzero((g != w).any(1))[0]
    if len(bad) and "geomID" in got.dtype.names:
        tie = (got["tfar"][bad].view(np.uint32) == want["tfar"][bad].view(np.uint32)) & (got["geomID"][bad] != NO_HIT) & (want["geomID"][bad] != NO_HIT)
        assert tie.all(), (f"{what}: {int((~tie).sum())} records differ beyond ties, first at {bad[~tie][:8].tolist()}", got[bad[~tie][:2]], want[bad[~tie][:2]])
    else:
        assert len(bad) == 0, (f"{what}: {len(bad)} records differ", got[bad[:2]], want[bad[:2]])
    assert len(bad) <= max_ties, (what, len(bad))


# ---- the reference's stored answers and the oracle ----------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("quality", [RTC_BUILD_QUALITY_LOW, RTC_BUILD_QUALITY_MEDIUM])
def test_golden_every_entry_point(b200, quality):
    """tutorials/instanced_geometry through all eight entry points, packets included, against the reference's outputs."""
    lib, dev = b200
    g = load_golden_instances()
    top, child, keep = traversal(lib, build_instanced, lib, dev, g, quality)
    assert lib.scene_device_traversable(top).nodes is None and lib.rtcGetDeviceError(dev) == 3   # the instance-traversal path was taken
    want = g["intersect_out"]
    for mode in MODES:
        got = lib.intersect(top, g["rays_in"].copy(), mode)
        rep = assert_parity(want, got)
        assert rep["ng_bit_exact"], (mode, rep)
        assert (got["instPrimID"] == want["instPrimID"]).all(), mode
        occ = lib.occluded(top, rays_of(g["rays_in"]), mode)
        assert (occ["tfar"].view(np.uint32) == g["occluded_out"]["tfar"].view(np.uint32)).all(), mode
    assert np.array_equal(bounds(lib, top), g["bounds"])
    lib.rtcReleaseScene(top)
    lib.rtcReleaseScene(child)


def _many_instances(rng, n, mesh_n):
    v, t = scenes.triangle_sphere(mesh_n)
    xf = []
    for i in range(n):
        q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        s = rng.uniform(0.3, 2.0, 3) * (1 if i % 5 else -1)
        m = (q * s).astype(np.float32)
        xf.append(np.concatenate([m.T.reshape(-1), rng.uniform(-20, 20, 3)]).astype(np.float32))
    return v, t, xf


@pytest.mark.gpu
def test_many_instances_vs_oracle(b200, oracle):
    """The 400 instances of test_instances_many_vs_oracle (mirrored and anisotropic transforms) against the oracle's two-level traversal."""
    lib, dev = b200
    rng = np.random.RandomState(21)
    v, t, xf = _many_instances(rng, 400, 40)
    g = dict(child=[(v, t, 0, 0xFFFFFFFF)], top=[], xfms=np.stack(xf), inst_masks=np.full(400, 0xFFFFFFFF, np.uint32), first_inst=0)
    top, child, keep = traversal(lib, build_instanced, lib, dev, g)
    org = rng.uniform(-25, 25, (200000, 3)).astype(np.float32)
    d = rng.normal(size=(200000, 3)).astype(np.float32)
    rays = make_rayhits(org, d)
    got = lib.intersect(top, rays.copy(), "1M")
    oc = oracle.scene(g["child"])
    ot = oracle.scene([], instances=[(oc, m, i, 0xFFFFFFFF) for i, m in enumerate(xf)])
    want = ot.trace(rays.copy(), nthreads=16)
    rep = compare_hits(want, got, TOL)
    assert rep["hits"] > 20000 and rep["id_mismatch"] == 0, rep

    def one_tri_instanced(g_, p_, i_):
        c = oracle.scene([(v, t[p_:p_ + 1], 0, 0xFFFFFFFF)])
        return oracle.scene([], instances=[(c, xf[i_], i_, 0xFFFFFFFF)])
    lost, unexplained = explain_hit_miss(oracle, rays, want, got, one_tri_instanced)
    assert lost == 0 and unexplained == 0, (rep, lost, unexplained)
    assert rep["max_rel_t"] <= TOL and rep["max_abs_uv"] <= TOL and rep["ng_bit_exact"], rep
    occ = lib.occluded(top, rays_of(rays), "1M")
    assert ((occ["tfar"] == -np.inf) != (got["geomID"] != NO_HIT)).sum() == 0
    ot.free()
    oc.free()
    lib.rtcReleaseScene(top)
    lib.rtcReleaseScene(child)


@pytest.mark.gpu
def test_too_big_to_flatten(b200, oracle):
    """4096 instances of a 1.1 M-triangle sphere: 4.6 G records flattened, more than an 80 GB card holds.  The default threshold
    takes instance traversal by itself; hits on a 4096-ray sample equal the oracle's."""
    lib, dev = b200
    rng = np.random.RandomState(5)
    v, t, xf = _many_instances(rng, 4096, 750)
    assert len(t) >= 1_000_000
    g = dict(child=[(v, t, 0, 0xFFFFFFFF)], top=[], xfms=np.stack(xf), inst_masks=np.full(4096, 0xFFFFFFFF, np.uint32), first_inst=0)
    top, child, keep = build_instanced(lib, dev, g, RTC_BUILD_QUALITY_LOW)
    assert lib.scene_device_traversable(top).nodes is None and lib.rtcGetDeviceError(dev) == 3
    rays = make_rayhits(rng.uniform(-25, 25, (4096, 3)).astype(np.float32), rng.normal(size=(4096, 3)).astype(np.float32))
    got = lib.intersect(top, rays.copy(), "1M")
    oc = oracle.scene(g["child"])
    ot = oracle.scene([], instances=[(oc, m, i, 0xFFFFFFFF) for i, m in enumerate(xf)])
    want = ot.trace(rays.copy(), nthreads=16)
    rep = compare_hits(want, got, TOL)
    assert rep["hits"] > 1000 and rep["id_mismatch"] == 0, rep

    def one_tri_instanced(g_, p_, i_):
        c = oracle.scene([(v, t[p_:p_ + 1], 0, 0xFFFFFFFF)])
        return oracle.scene([], instances=[(c, xf[i_], i_, 0xFFFFFFFF)])
    lost, unexplained = explain_hit_miss(oracle, rays, want, got, one_tri_instanced)
    assert lost == 0 and unexplained == 0, (rep, lost, unexplained)
    ot.free()
    oc.free()
    lib.rtcReleaseScene(top)
    lib.rtcReleaseScene(child)


# ---- equal to flattening ---------------------------------------------------------------------------------------------------------
def _tops(lib, dev, child, own, insts, flags):
    """The same top-level scene twice, flattened and with instance traversal: `own` meshes (v, t, geomID, mask) and instances
    (xfm, mask, geomID) of `child`."""
    out, keep = [], []
    for force in (False, True):
        top = lib.rtcNewScene(dev)
        lib.rtcSetSceneFlags(top, flags)
        for (v, t, gid, mask) in own:
            keep.append(lib.add_triangle_mesh(dev, top, v, t, mask=mask, geom_id=gid)[1])
        for (m, mask, gid) in insts:
            lib.add_instance(dev, top, child, m, mask=int(mask), geom_id=gid)
        if force:
            traversal(lib, lib.rtcCommitScene, top)
        else:
            lib.rtcCommitScene(top)
        lib.check(dev)
        out.append(top)
    return out[0], out[1], keep


def _quads_instances(lib, dev, flags):
    """test_trace_schedules' quads_instances: a quad terrain under six rotations with instance masks, beside a triangle sphere"""
    vq, q = scenes.quad_terrain(64)
    vs, ts = scenes.triangle_sphere(40, center=(0.0, -1.2, 0.0), radius=0.5)
    rng = np.random.RandomState(2)
    insts = []
    for i, mask in enumerate((1, 2, 4, 3, 6, 0xFFFFFFFF)):
        m, _r = np.linalg.qr(rng.normal(size=(3, 3)))
        insts.append((np.concatenate([m[:, 0], m[:, 1], m[:, 2], rng.uniform(-1.5, 1.5, 3)]).astype(np.float32), mask, 1 + i))
    child, keep = build_scene(lib, dev, [(vq, q, 0, 0xFFFFFFFF)], flags=flags)
    flat, inst, k2 = _tops(lib, dev, child, [(vs, ts, 0, 0xFFFFFFFF)], insts, flags)
    return flat, inst, [child], [keep, k2], ((0, 0, 0), 4.0, (0.2, 0.5, -5.0), (0.0, -0.1, 1.0), 3)


def _hair_instances(lib, dev, flags):
    """test_trace_schedules' hair_instances: every curve and point kind around a sphere, under six transforms with instance masks"""
    S = instanced_hair_scene()
    top0, child, keep = build_instanced_hair(lib, dev, S)
    lib.rtcReleaseScene(top0)
    flat, inst, k2 = _tops(lib, dev, child, [], [(m, S["masks"][i], i) for i, m in enumerate(S["xfms"])], flags)
    return flat, inst, [child], [keep, k2, S], ((0, 0, 0), 4.0, (0.0, 0.3, -7.0), (0.0, 0.0, 1.0), 5)


EQUAL_SCENES = {"quads_instances": _quads_instances, "hair_instances": _hair_instances}


@pytest.mark.gpu
@pytest.mark.parametrize("robust", [False, True])
@pytest.mark.parametrize("scene", list(EQUAL_SCENES))
def test_equal_to_flattening(b200, scene, robust):
    """The same scene committed flattened and with instance traversal writes the same bytes for every ray through every entry point:
    batched host and device, packets, any hit, the counting kernels and the fused gather."""
    import torch
    lib, dev = b200
    flat, inst, children, keep, (center, radius, eye, look, seed) = EQUAL_SCENES[scene](lib, dev, 4 if robust else 0)
    assert lib.scene_device_traversable(flat).nodes is not None
    rays = ray_mix(lib, dev, flat, center, radius, eye, look, seed=seed)
    ties = len(rays) // 1000
    want = lib.intersect(flat, rays.copy(), "1M")
    assert (want["geomID"] != NO_HIT).sum() > len(rays) // 20
    same_but_ties(lib.intersect(inst, rays.copy(), "1M"), want, "1M", ties)
    for mode in ("4M", "8M", "16M"):
        same_but_ties(lib.intersect(inst, rays.copy(), mode), lib.intersect(flat, rays.copy(), mode), mode, ties)
    for mode in ("1M", "4M", "16M"):
        same_but_ties(lib.occluded(inst, rays_of(rays), mode), lib.occluded(flat, rays_of(rays), mode), "occluded " + mode, 0)
    # device entry point and the counting kernels
    for sc in (inst, flat):
        lib.rtcb200SetSceneStatCounters(sc, 1)
        lib.rtcb200ResetSceneStatCounters(sc)
    buf_i, buf_f = _cuda(rays), _cuda(rays)
    a = lib.args()
    lib.rtcb200Intersect1MDevice(inst, C.c_void_p(buf_i.data_ptr()), len(rays), C.byref(a), _stream())
    lib.rtcb200Intersect1MDevice(flat, C.c_void_p(buf_f.data_ptr()), len(rays), C.byref(a), _stream())
    torch.cuda.synchronize()
    lib.check(dev)
    same_but_ties(buf_i.cpu().numpy().view(RAYHIT_DTYPE), buf_f.cpu().numpy().view(RAYHIT_DTYPE), "1MDevice, counting", ties)
    st = lib.scene_stats(inst)
    assert st.trav_rays == len(rays) and st.trav_nodes > 0 and st.trav_tris > 0, (st.trav_rays, st.trav_nodes, st.trav_tris)
    for sc in (inst, flat):
        lib.rtcb200SetSceneStatCounters(sc, 0)
    # fused gather: one 32-byte record per ray, in both gather modes
    for mode in (0, 1):
        with tuning(lib, gather_mode=mode):
            outs = []
            for sc in (inst, flat):
                buf = _cuda(rays)
                rec = torch.zeros(len(rays) * 8, dtype=torch.float32, device="cuda")
                lib.rtcb200Intersect1MGatherDevice(sc, C.c_void_p(buf.data_ptr()), len(rays), C.byref(a), _stream(), C.c_void_p(rec.data_ptr()))
                torch.cuda.synchronize()
                lib.check(dev)
                outs.append((buf.cpu().numpy().view(RAYHIT_DTYPE), rec.cpu().numpy().reshape(-1, 8)))
            same_but_ties(outs[0][0], outs[1][0], f"gather {mode}", ties)
            same = (outs[0][1].view(np.uint32) == outs[1][1].view(np.uint32)).all(1)
            assert (~same).sum() <= ties, (mode, int((~same).sum()))
    b_flat, b_inst = bounds(lib, flat), bounds(lib, inst)
    assert np.array_equal(b_flat, b_inst), (b_flat, b_inst)
    lib.rtcReleaseScene(inst)
    lib.rtcReleaseScene(flat)
    for c in children:
        lib.rtcReleaseScene(c)


@pytest.mark.gpu
def test_interpolation_on_instance_traversal(b200):
    """Batched interpolation keys on instID and geomID: hits of the instance-traversal scene interpolate as the flattened scene's do."""
    lib, dev = b200
    flat, inst, children, keep, (center, radius, eye, look, seed) = _quads_instances(lib, dev, 0)
    rays = ray_mix(lib, dev, flat, center, radius, eye, look, seed=seed)
    hf, hi = lib.intersect(flat, rays.copy(), "1M"), lib.intersect(inst, rays.copy(), "1M")
    same = (np.ascontiguousarray(hf).view(np.uint8).reshape(len(hf), -1) == np.ascontiguousarray(hi).view(np.uint8).reshape(len(hi), -1)).all(1)
    hit = same & (hf["geomID"] != NO_HIT)
    assert hit.sum() > 1000
    pf = lib.interpolate_hits(flat, hf[hit].copy(), RTC_BUFFER_TYPE_VERTEX, 0, 3)
    pi = lib.interpolate_hits(inst, hi[hit].copy(), RTC_BUFFER_TYPE_VERTEX, 0, 3)
    lib.check(dev)
    for n in pf:
        assert np.array_equal(pf[n].view(np.uint32), pi[n].view(np.uint32)), n
        assert np.isfinite(pi[n]).all(), n
    lib.rtcReleaseScene(inst)
    lib.rtcReleaseScene(flat)
    for c in children:
        lib.rtcReleaseScene(c)


# ---- API, masks, edits ---------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_masks_moves_and_child_release(b200):
    """Instance masks, moving an instance, and tracing after the application released the instanced scene."""
    lib, dev = b200
    v, t = scenes.triangle_sphere(8)
    child, keep = build_scene(lib, dev, [(v, t, 0, 0xFFFFFFFF)])
    top = lib.rtcNewScene(dev)
    col = np.array([2, 0, 0, 0, 2, 0, 0, 0, 2, 5, 6, 7], np.float32)
    g = lib.rtcGetGeometry(top, lib.add_instance(dev, top, child, col))
    traversal(lib, lib.rtcCommitScene, top)
    lib.check(dev)
    out = lib.intersect(top, make_rayhits([[5, 6, 0]], [[0, 0, 1]]), "1")
    assert out["geomID"][0] == 0 and out["instID"][0] == 0 and out["instPrimID"][0] == 0 and abs(out["tfar"][0] - 5.0) < 1e-5, out
    col[9:] = (0, 0, 10)
    lib.rtcSetGeometryTransform(g, 0, RTC_FORMAT_FLOAT3X4_COLUMN_MAJOR, _ptr(col))
    lib.rtcCommitGeometry(g)
    traversal(lib, lib.rtcCommitScene, top)
    out = lib.intersect(top, make_rayhits([[0, 0, 0]], [[0, 0, 1]]), "1")
    assert abs(out["tfar"][0] - 8.0) < 1e-5 and out["instID"][0] == 0
    lib.rtcSetGeometryMask(g, 0x4)
    lib.rtcCommitGeometry(g)
    traversal(lib, lib.rtcCommitScene, top)
    for mode in ("1", "1M", "8M"):
        assert lib.intersect(top, make_rayhits([[0, 0, 0]], [[0, 0, 1]], mask=0x3), mode)["geomID"][0] == NO_HIT, mode
        assert lib.intersect(top, make_rayhits([[0, 0, 0]], [[0, 0, 1]], mask=0x4), mode)["geomID"][0] == 0, mode
        occ = lib.occluded(top, rays_of(make_rayhits([[0, 0, 0]], [[0, 0, 1]], mask=0x3)), mode)
        assert occ["tfar"][0] != -np.inf, mode
    lib.rtcReleaseScene(child)   # the instance keeps it alive; the scene's own copy of its BVH is traced
    assert lib.intersect(top, make_rayhits([[0, 0, 0]], [[0, 0, 1]], mask=0x4), "1")["geomID"][0] == 0
    lib.check(dev)
    lib.rtcReleaseScene(top)


@pytest.mark.gpu
def test_child_recommit_and_moves_rebuild_no_child_bvh(b200, capfd):
    """A child re-commit reaches the instances at the parent's next commit, and not before; moving instances rebuilds only the top
    level (the verbose commit log counts the instanced scenes' BVHs built by each commit)."""
    from embree_b200.rtc import RTC_BUFFER_TYPE_INDEX, RTC_FORMAT_FLOAT3, RTC_FORMAT_UINT3, RTC_GEOMETRY_TYPE_TRIANGLE
    lib, _ = b200
    dev = lib.new_device("verbose=2")
    v, t = scenes.triangle_sphere(10)
    vpad = np.zeros(v.size + 4, np.float32)
    vpad[:v.size] = v.ravel()
    g = lib.rtcNewGeometry(dev, RTC_GEOMETRY_TYPE_TRIANGLE)
    lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, _ptr(vpad), 0, 12, len(v))
    lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT3, _ptr(t), 0, 12, len(t))
    lib.rtcCommitGeometry(g)
    child = lib.rtcNewScene(dev)
    lib.rtcAttachGeometry(child, g)
    lib.rtcCommitScene(child)
    top = lib.rtcNewScene(dev)
    insts = []
    for k in range(16):
        col = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 3 * k, 0, 10], np.float32)
        insts.append((lib.rtcGetGeometry(top, lib.add_instance(dev, top, child, col)), col))
    capfd.readouterr()
    traversal(lib, lib.rtcCommitScene, top)
    lib.check(dev)
    log = capfd.readouterr().err
    assert re.search(r"commit \(instance traversal\): 16 instances of 1 scenes, 1 rebuilt", log), log
    r = make_rayhits([[0, 0, 0]], [[0, 0, 1]])
    assert abs(lib.intersect(top, r.copy(), "1")["tfar"][0] - 9.0) < 1e-5
    vpad[:v.size] *= 2.0
    lib.rtcUpdateGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0)
    lib.rtcCommitGeometry(g)
    lib.rtcCommitScene(child)
    assert abs(lib.intersect(top, r.copy(), "1")["tfar"][0] - 9.0) < 1e-5   # the parent still traces what it committed
    capfd.readouterr()
    traversal(lib, lib.rtcCommitScene, top)
    lib.check(dev)
    assert re.search(r"16 instances of 1 scenes, 1 rebuilt", capfd.readouterr().err)
    out = lib.intersect(top, r.copy(), "1")
    assert abs(out["tfar"][0] - 8.0) < 1e-5 and out["instID"][0] == 0, out
    for step, moved in enumerate(([0], list(range(16)))):   # move one instance, then all of them
        for k in moved:
            gk, col = insts[k]
            col[11] += 1.0
            lib.rtcSetGeometryTransform(gk, 0, RTC_FORMAT_FLOAT3X4_COLUMN_MAJOR, _ptr(col))
            lib.rtcCommitGeometry(gk)
        capfd.readouterr()
        traversal(lib, lib.rtcCommitScene, top)
        lib.check(dev)
        log = capfd.readouterr().err
        assert re.search(r"16 instances of 1 scenes, 0 rebuilt", log), (step, log)
        assert abs(lib.intersect(top, r.copy(), "1")["tfar"][0] - (8.0 + step + 1)) < 1e-5
    lib.rtcReleaseGeometry(g)
    lib.rtcReleaseScene(child)
    lib.rtcReleaseScene(top)
    lib.rtcReleaseDevice(dev)


@pytest.mark.gpu
def test_selection_and_refusals(b200, capfd):
    """The commit log names the path; the default flattens the small golden scene.  Host filter callbacks and device-side queries
    refuse instance-traversal scenes with RTC_ERROR_INVALID_OPERATION instead of tracing them some other way."""
    from embree_b200.rtc import FILTER_FUNCTION
    lib, _ = b200
    dev = lib.new_device("verbose=2")
    g = load_golden_instances()
    capfd.readouterr()
    flat, child, keep = build_instanced(lib, dev, g)
    assert "commit (instances flattened)" in capfd.readouterr().err
    inst, child2, keep2 = traversal(lib, build_instanced, lib, dev, g)
    assert "commit (instance traversal)" in capfd.readouterr().err
    assert lib.scene_device_traversable(flat).nodes is not None
    lib.check(dev)
    lib.scene_device_traversable(inst)
    assert lib.rtcGetDeviceError(dev) == 3

    @FILTER_FUNCTION
    def accept(args):
        pass
    a = lib.args(filter=accept, invoke_argument_filter=True)
    rays = g["rays_in"].copy()
    lib.intersect(inst, rays, "1M", args=a)
    assert lib.rtcGetDeviceError(dev) == 3
    lib.intersect(flat, g["rays_in"].copy(), "1M", args=a)
    lib.check(dev)
    for sc in (flat, inst, child, child2):
        lib.rtcReleaseScene(sc)
    lib.rtcReleaseDevice(dev)


@pytest.mark.gpu
@pytest.mark.parametrize("robust", [False, True])
def test_general_scene_equal_to_flattening(b200, robust):
    """test_bvh_structure's general scene (triangle meshes with strides, quads, every curve and point kind, and instances of a child
    holding triangles, quads, round curves and points) writes the same records on both paths."""
    from tests.test_bvh_structure import build_general_scene
    lib, dev = b200
    flat, _, keep_f = build_general_scene(lib, dev, robust, RTC_BUILD_QUALITY_MEDIUM)
    inst, _, keep_i = traversal(lib, build_general_scene, lib, dev, robust, RTC_BUILD_QUALITY_MEDIUM)
    assert lib.scene_device_traversable(flat).nodes is not None
    lib.scene_device_traversable(inst)
    assert lib.rtcGetDeviceError(dev) == 3
    rays = ray_mix(lib, dev, flat, (0, 0, -1), 6.0, (0.0, 0.5, -12.0), (0.0, 0.0, 1.0), seed=11)
    ties = len(rays) // 1000
    for mode in ("1M", "8M"):
        same_but_ties(lib.intersect(inst, rays.copy(), mode), lib.intersect(flat, rays.copy(), mode), mode, ties)
    same_but_ties(lib.occluded(inst, rays_of(rays), "1M"), lib.occluded(flat, rays_of(rays), "1M"), "occluded", 0)
    assert np.array_equal(bounds(lib, flat), bounds(lib, inst))
    for sc, keep in ((inst, keep_i), (flat, keep_f)):
        lib.rtcReleaseScene(sc)
        lib.rtcReleaseScene(keep[-1])


@pytest.mark.gpu
def test_geometry_getters_on_instance_traversal(b200):
    """rtcGetGeometryTransform and rtcGetGeometryUserData answer for the instances of an instance-traversal scene."""
    lib, dev = b200
    v, t = scenes.triangle_sphere(8)
    child, keep = build_scene(lib, dev, [(v, t, 0, 0xFFFFFFFF)])
    top = lib.rtcNewScene(dev)
    cols = [np.array([1, 0, 0, 0, 2, 0, 0, 0, 3, 4 * k, 1, 2], np.float32) for k in range(3)]
    ids = [lib.add_instance(dev, top, child, m) for m in cols]
    for k, i in enumerate(ids):
        lib.rtcSetGeometryUserData(lib.rtcGetGeometry(top, i), 1000 + k)
    traversal(lib, lib.rtcCommitScene, top)
    lib.check(dev)
    for k, i in enumerate(ids):
        back = np.zeros(12, np.float32)
        lib.rtcGetGeometryTransform(lib.rtcGetGeometry(top, i), 0.0, RTC_FORMAT_FLOAT3X4_COLUMN_MAJOR, _ptr(back))
        assert np.array_equal(back, cols[k]), (k, back)
        assert lib.rtcGetGeometryUserData(lib.rtcGetGeometry(top, i)) == 1000 + k
        out = lib.intersect(top, make_rayhits([[4 * k, 1, -10]], [[0, 0, 1]]), "1")
        assert out["instID"][0] == i and out["geomID"][0] == 0, (k, out)
    lib.check(dev)
    lib.rtcReleaseScene(top)
    lib.rtcReleaseScene(child)


@pytest.mark.gpu
def test_large_scenes_keep_filters_and_device_queries_at_the_default(b200, capfd):
    """17 instances of a 1 M-triangle sphere (17 M flattened records) are flattened at the shipped tuning and keep the device-side
    queries; with an intersect filter on the instanced mesh the scene is flattened even when the threshold asks for instance traversal,
    and the callback is called."""
    from embree_b200.rtc import FILTER_FUNCTION
    lib, _ = b200
    dev = lib.new_device("verbose=2")
    v, t = scenes.triangle_sphere(500)
    child, keep = build_scene(lib, dev, [(v, t, 0, 0xFFFFFFFF)])
    xf = []
    rng = np.random.RandomState(3)
    for k in range(17):
        xf.append(np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 3 * k, 0, rng.uniform(0, 1)], np.float32))

    def top_scene(force):
        top = lib.rtcNewScene(dev)
        for m in xf:
            lib.add_instance(dev, top, child, m)
        capfd.readouterr()
        if force:
            traversal(lib, lib.rtcCommitScene, top)
        else:
            lib.rtcCommitScene(top)
        lib.check(dev)
        return top, capfd.readouterr().err
    top, log = top_scene(False)
    assert "commit (instances flattened)" in log, log
    assert lib.scene_device_traversable(top).nodes is not None
    lib.check(dev)
    rays = make_rayhits([[3 * k, 0, -10] for k in range(17)], [[0, 0, 1]] * 17)
    plain = lib.intersect(top, rays.copy(), "1M")
    assert (plain["geomID"] == 0).all()
    lib.rtcReleaseScene(top)
    calls = []

    def reject(args):
        a = args.contents
        calls.append(a.N)
        for lane in range(a.N):
            a.valid[lane] = 0
    fn = FILTER_FUNCTION(reject)
    g = lib.rtcGetGeometry(child, 0)
    lib.rtcSetGeometryIntersectFilterFunction(g, fn)
    for force in (False, True):
        top, log = top_scene(force)
        assert "commit (instances flattened)" in log, (force, log)
        calls.clear()
        out = lib.intersect(top, rays.copy(), "1M")
        lib.check(dev)
        assert calls and (out["geomID"] == NO_HIT).all(), (force, len(calls))
        lib.rtcReleaseScene(top)
    lib.rtcSetGeometryIntersectFilterFunction(g, None)
    lib.rtcReleaseScene(child)
    lib.rtcReleaseDevice(dev)
