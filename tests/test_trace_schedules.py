"""A ray's record must not depend on how the trace kernel schedules it.

trace.cu's persistent warps decide at run time when a warp refills, when it runs a triangle or curve step and which rays share a
warp; the SPREAD step (the warp-wide triangle test) may split one ray's triangles over several steps when its 32-slot queue
overflows.  None of this may change a result: every record (all 96 bytes of an RTCRayHit, all 48 of an RTCRay) must equal the one
the shipped tuning writes through rtcb200Intersect1MDevice / rtcb200Occluded1MDevice, for a permuted or reversed ray order, every
rtcb200SetTuning knob of the trace kernels and the host pipeline set one at a time, the packet entry points with a random valid
mask, the host-pointer pipeline, the fused hit gather and the counting kernels -- over a scene of each kind the kernel is
instantiated for.  The ray origins of the signed-zero stream lie exactly on a planar grid, so every ray meets several candidates at
t = +0 or -0 and the winner among equal distances decides the record.

Only "tri_spread" 0 (the per-lane closest-hit triangle test) uses another acceptance rule; it is held to the SPREAD kernel by
distance and to the filter-callback kernel, which runs the same per-lane rule, byte for byte."""
import contextlib
import ctypes as C
import os
import re

import numpy as np
import pytest

from embree_b200 import scenes
from embree_b200.rtc import FILTER_FUNCTION, RAY_DTYPE, RAYHIT_DTYPE, aligned_empty, from_packets, packet_dtype, rays_of, to_packets
from tests import bvh_check
from tests.parity import (build_instanced_hair, compare_hits, instanced_hair_scene, load_oracle, signed_zero_grid,
                          zero_distance_candidates)
from tests.test_device_traversal import query_rays
from tests.test_gpu_parity import _dynamic_meshes, build_instanced, build_scene

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "embree_b200", "csrc")


# ---- tuning ------------------------------------------------------------------------------------------------------------------
def shipped_tuning():
    """The shipped value of every rtcb200SetTuning key, read from the source: the members of struct Tuning (rtk_device.h) and the
    host pipeline's g_host_* settings (rtcore_shim.cpp).  There is no getter; parsing keeps these from drifting from the source."""
    with open(os.path.join(CSRC, "rtk_device.h")) as f:
        body = re.search(r"struct Tuning \{(.*?)\n\};", f.read(), re.S).group(1)
    out = {}
    for line in body.splitlines():
        m = re.match(r"\s*int\s+([^;]*);", line.split("//")[0])
        for part in (m.group(1).split(",") if m else []):
            k, v = part.split("=")
            out[k.strip()] = int(v)
    with open(os.path.join(CSRC, "rtcore_shim.cpp")) as f:
        shim = f.read()
    for key in ("host_chunk_log2", "host_streams", "host_d2h_partial"):
        out[key] = int(re.search(r"\bg_%s = (-?\d+)" % key, shim).group(1))
    assert {"tri_batch_min", "tri_wait_max", "refill_min", "blocks_per_sm", "tri_spread", "gather_mode"} <= set(out), out
    return out


SHIPPED = shipped_tuning()


@contextlib.contextmanager
def tuning(lib, **keys):
    """Set rtcb200SetTuning keys for the body; every key is back at its shipped value afterwards, whatever happened."""
    try:
        for k, v in keys.items():
            assert lib.rtcb200SetTuning(k.encode(), int(v)) == 0, (k, v)
        yield
    finally:
        for k, v in SHIPPED.items():
            assert lib.rtcb200SetTuning(k.encode(), v) == 0, k


# ---- tracing and comparing -------------------------------------------------------------------------------------------------
def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).cuda()


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def trace_device(lib, dev, sc, recs, occluded=False, args=None):
    """rtcb200Intersect1MDevice / rtcb200Occluded1MDevice on a device copy of `recs`; returns the records it left."""
    import torch
    buf = _cuda(recs)
    a = args if args is not None else lib.args()
    fn = lib.rtcb200Occluded1MDevice if occluded else lib.rtcb200Intersect1MDevice
    fn(sc, C.c_void_p(buf.data_ptr()), len(recs), C.byref(a), _stream())
    torch.cuda.synchronize()
    lib.check(dev)
    return buf.cpu().numpy().view(RAY_DTYPE if occluded else RAYHIT_DTYPE)


def host_copy(recs):
    out = aligned_empty(len(recs), recs.dtype)
    out[:] = recs
    return out


def assert_same_records(got, want, what):
    g = np.ascontiguousarray(got).view(np.uint8).reshape(len(got), -1)
    w = np.ascontiguousarray(want).view(np.uint8).reshape(len(want), -1)
    assert g.shape == w.shape, (what, g.shape, w.shape)
    bad = np.nonzero((g != w).any(1))[0]
    assert len(bad) == 0, (f"{what}: {len(bad)} of {len(want)} records differ, first at {bad[:8].tolist()}",
                           got[bad[:2]], want[bad[:2]])


# ---- scenes --------------------------------------------------------------------------------------------------------------------
class Case:
    """A committed scene, its rays and the baseline: what the shipped tuning writes for them through the Device entry points."""

    def __init__(self, lib, dev, sc, keep, release, rays, general, curves=0, oracle_meshes=None, robust=False):
        self.lib, self.dev, self.sc, self.keep, self.release = lib, dev, sc, keep, release
        self.rh, self.general, self.curves = rays, general, curves
        self.oracle_meshes, self.robust = oracle_meshes, robust
        t = lib.scene_device_traversable(sc)
        lib.check(dev)
        assert (t.general, t.curves) == (general, curves), (t.general, t.curves)
        self.ray = rays_of(rays)
        self.base_i = trace_device(lib, dev, sc, rays)
        self.base_o = trace_device(lib, dev, sc, self.ray, occluded=True)
        hit = self.base_i["geomID"] != 0xFFFFFFFF
        assert hit.sum() > len(rays) // 20 and (~hit).sum() > 0, hit.sum()
        assert ((self.base_o["tfar"] == -np.inf) == hit).all()   # occluded agrees with intersect on every ray


def ray_mix(lib, dev, sc, center, radius, eye, look, seed, n_query=40007, camera=(160, 120), n_bounce=30011):
    """Incoherent rays with every case query_rays covers (masks, tnear windows, tfar < 0, zero direction components), coherent
    camera rays and diffuse bounces off the camera rays' hits, in one stream whose length is not a multiple of 32."""
    import torch
    q = query_rays(n_query, center, radius, seed=seed)
    cam = scenes.as_numpy_rayhits(scenes.primary_rays(camera[0], camera[1], eye=eye, look=look))
    traced = trace_device(lib, dev, sc, cam)
    hits = torch.from_numpy(traced.view(np.float32).reshape(-1, 24).copy())
    bounce = scenes.as_numpy_rayhits(scenes.diffuse_bounce_rays(hits, seed=seed, replicate=2))[:n_bounce]
    rays = aligned_empty(len(q) + len(cam) + len(bounce), RAYHIT_DTYPE)
    rays[:len(q)], rays[len(q):len(q) + len(cam)], rays[len(q) + len(cam):] = q, cam, bounce
    rays["id"] = np.arange(len(rays), dtype=np.uint32)
    if len(rays) % 32 == 0:
        rays = host_copy(rays[:-1])
    return rays


def _sphere(lib, dev, robust):
    v, t = scenes.triangle_sphere(200)
    v2, t2 = scenes.triangle_sphere(60, center=(0.3, 0.2, -0.1), radius=0.4)
    meshes = [(v, t, 0, 1), (v2, t2, 1, 2)]
    sc, keep = build_scene(lib, dev, meshes, flags=4 if robust else 0)
    rays = ray_mix(lib, dev, sc, (0, 0, 0), 2.0, (0.1, 0.2, -3.0), (0.0, 0.0, 1.0), seed=1)
    return Case(lib, dev, sc, keep, [sc], rays, 0, oracle_meshes=meshes, robust=robust)


def _quads_instances(lib, dev):
    vq, q = scenes.quad_terrain(64)
    vs, ts = scenes.triangle_sphere(40, center=(0.0, -1.2, 0.0), radius=0.5)
    rng = np.random.RandomState(2)
    xfms = []
    for _ in range(6):
        m, _r = np.linalg.qr(rng.normal(size=(3, 3)))
        xfms.append(np.concatenate([m[:, 0], m[:, 1], m[:, 2], rng.uniform(-1.5, 1.5, 3)]).astype(np.float32))
    g = dict(child=[(vq, q, 0, 0xFFFFFFFF)], top=[(vs, ts, 0, 0xFFFFFFFF)], xfms=xfms,
             inst_masks=np.array([1, 2, 4, 3, 6, 0xFFFFFFFF], np.uint32), first_inst=1)
    top, child, keep = build_instanced(lib, dev, g)
    rays = ray_mix(lib, dev, top, (0, 0, 0), 4.0, (0.2, 0.5, -5.0), (0.0, -0.1, 1.0), seed=3)
    return Case(lib, dev, top, keep, [top, child], rays, 1)


def _hair_instances(lib, dev):
    S = instanced_hair_scene()
    top, child, keep = build_instanced_hair(lib, dev, S)
    rays = ray_mix(lib, dev, top, (0, 0, 0), 4.0, (0.0, 0.3, -7.0), (0.0, 0.0, 1.0), seed=5, n_query=20011, camera=(128, 96), n_bounce=15013)
    return Case(lib, dev, top, [keep, S], [top, child], rays, 1, curves=2)


def _points(lib, dev):
    rng = np.random.RandomState(6)
    sc = lib.rtcNewScene(dev)
    keep = []
    for k, kind in enumerate(("sphere", "disc", "oriented_disc")):
        pv = np.concatenate([rng.normal(size=(20000, 3)), rng.uniform(0.005, 0.03, (20000, 1))], 1).astype(np.float32)
        nrm = rng.normal(size=(20000, 3)).astype(np.float32)
        keep.append(lib.add_points(dev, sc, pv, kind, normals=nrm if kind == "oriented_disc" else None, mask=1 << k)[1])
    lib.rtcCommitScene(sc)
    lib.check(dev)
    rays = ray_mix(lib, dev, sc, (0, 0, 0), 3.0, (0.0, 0.0, -5.0), (0.0, 0.0, 1.0), seed=7)
    return Case(lib, dev, sc, keep, [sc], rays, 1, curves=1)


def _dynamic(lib, dev):
    """An RTC_SCENE_FLAG_DYNAMIC scene re-committed after one mesh was rebuilt and one refitted: the two-level assembly."""
    from embree_b200.rtc import RTC_BUFFER_TYPE_VERTEX
    meshes = _dynamic_meshes(24)
    sc = lib.rtcNewScene(dev)
    lib.rtcSetSceneFlags(sc, 1)
    bufs = [lib.add_triangle_mesh(dev, sc, v, t, mask=0xFFFFFFFF, quality=3 if i == 5 else None)[1] for i, (v, t) in enumerate(meshes)]
    lib.rtcCommitScene(sc)
    for i, builder in ((2, 3), (5, None)):   # mesh 2 moves: the commit assembles the kept per-mesh BVHs; then mesh 5 is refitted
        if i == 2:
            bufs[i][0][:meshes[i][0].size] += np.float32(0.35)
        else:
            bufs[i][0][:meshes[i][0].size] *= np.float32(1.1)
        g = lib.rtcGetGeometry(sc, i)
        lib.rtcUpdateGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0)
        lib.rtcCommitGeometry(g)
        lib.rtcCommitScene(sc)
        lib.check(dev)
        assert builder is None or lib.scene_stats(sc).builder == builder
    cur = [(bufs[i][0][:meshes[i][0].size].reshape(-1, 3).copy(), meshes[i][1], i, 0xFFFFFFFF) for i in range(len(meshes))]
    rays = ray_mix(lib, dev, sc, (0, 0, 0), 5.0, (0.5, 0.5, -9.0), (0.0, 0.0, 1.0), seed=8)
    return Case(lib, dev, sc, bufs, [sc], rays, 0, oracle_meshes=cur)


def _terrain(lib, dev):
    """A fine terrain seen by coherent camera rays at a low angle: every leaf node the rays reach holds many triangles, so the
    SPREAD step's 32-slot queue overflows and one ray's triangles are split over several steps."""
    v, t = scenes.terrain(384)
    meshes = [(v, t, 0, 0xFFFFFFFF)]
    sc, keep = build_scene(lib, dev, meshes)
    rays = ray_mix(lib, dev, sc, (0, 0, 0), 1.5, (0.0, 0.8, -1.2), (0.0, -0.6, 1.0), seed=9, n_query=20011, camera=(256, 192))
    return Case(lib, dev, sc, keep, [sc], rays, 0, oracle_meshes=meshes)


BUILDERS = {
    "sphere": lambda L, d: _sphere(L, d, False),         # GENERAL 0: SPREAD for closest and any hit
    "sphere_robust": lambda L, d: _sphere(L, d, True),   # per-lane Pluecker test
    "quads_instances": _quads_instances,                 # GENERAL 1
    "hair_instances": _hair_instances,                   # GENERAL 2 with curves: the curve_* knobs
    "points": _points,                                   # GENERAL 2, points only: the point_* knobs
    "dynamic": _dynamic,                                 # two-level assembly after a rebuild and a refit
    "terrain": _terrain,                                 # dense leaves: SPREAD queue overflow
}
SCENES = list(BUILDERS)


@pytest.fixture(scope="module")
def cases(b200):
    lib, dev = b200
    built = {}

    def get(name):
        if name not in built:
            built[name] = BUILDERS[name](lib, dev)
        return built[name]
    yield get
    for c in built.values():
        for s in c.release:
            lib.rtcReleaseScene(s)


# ---- the baseline against the oracle ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("scene", [s for s in SCENES if s in ("sphere", "sphere_robust", "dynamic", "terrain")])
def test_baseline_matches_the_oracle(cases, scene):
    """The records every variant below is held to are right: hits equal the C oracle's over the same triangles."""
    c = cases(scene)
    want = load_oracle().scene(c.oracle_meshes, robust=c.robust).trace(host_copy(c.rh), nthreads=8)
    rep = compare_hits(want, c.base_i, 1e-4, meshes=c.oracle_meshes)
    assert rep["id_mismatch"] == 0 and rep["hit_miss_disagree"] == 0 and rep["tie"] <= 50, rep
    assert rep["max_rel_t"] <= 1e-4 and rep["max_abs_uv"] <= 1e-4 and rep["miss_untouched"], rep


# ---- ray order ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", ["permuted", "reversed"])
@pytest.mark.parametrize("scene", SCENES)
def test_ray_order(cases, scene, order):
    """Other rays in the warp, the same record: the stream is traced in another order and put back."""
    c = cases(scene)
    n = len(c.rh)
    perm = np.random.RandomState(12).permutation(n) if order == "permuted" else np.arange(n)[::-1]
    got_i, got_o = aligned_empty(n, RAYHIT_DTYPE), aligned_empty(n, RAY_DTYPE)
    got_i[perm] = trace_device(c.lib, c.dev, c.sc, host_copy(c.rh[perm]))
    got_o[perm] = trace_device(c.lib, c.dev, c.sc, host_copy(c.ray[perm]), occluded=True)
    assert_same_records(got_i, c.base_i, "intersect")
    assert_same_records(got_o, c.base_o, "occluded")


# ---- the trace kernel's knobs, one at a time -------------------------------------------------------------------------------
KNOBS = {
    "tri_step_1_0": dict(tri_batch_min=1, tri_wait_max=0),          # a triangle step whenever one lane has a triangle
    "tri_step_32_1000": dict(tri_batch_min=32, tri_wait_max=1000),  # ... only when every lane has one or none has a node
    "refill_1": dict(refill_min=1),
    "refill_32": dict(refill_min=32),                               # refill only when the whole warp is idle
    "blocks_per_sm_1": dict(blocks_per_sm=1),                       # each warp walks many 32-ray blocks
    "curve_step_1_0": dict(curve_batch_min=1, curve_wait_max=0),
    "curve_step_32_1000": dict(curve_batch_min=32, curve_wait_max=1000),
    "curve_blocks_per_sm_1": dict(curve_blocks_per_sm=1),
    "point_step_1_0": dict(point_batch_min=1, point_wait_max=0),
    "point_step_32_1000": dict(point_batch_min=32, point_wait_max=1000),
    "no_tma": dict(use_tma=0),
    "no_occluded_spread": dict(tri_spread_occluded=0),              # the per-lane any-hit kernel
}


@pytest.mark.parametrize("knob", list(KNOBS))
@pytest.mark.parametrize("scene", SCENES)
def test_tuning_knob(cases, scene, knob):
    c = cases(scene)
    with tuning(c.lib, **KNOBS[knob]):
        got_i = trace_device(c.lib, c.dev, c.sc, c.rh)
        got_o = trace_device(c.lib, c.dev, c.sc, c.ray, occluded=True)
    assert_same_records(got_i, c.base_i, "intersect")
    assert_same_records(got_o, c.base_o, "occluded")


# ---- packets -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [4, 8, 16])
@pytest.mark.parametrize("scene", SCENES)
def test_packets(cases, scene, K):
    """rtcb200IntersectNMDevice / rtcb200OccludedNMDevice with a random valid mask: active lanes as the baseline, inactive lanes
    untouched."""
    import torch
    c = cases(scene)
    n = len(c.rh)
    for occluded, recs, base in ((False, c.rh, c.base_i), (True, c.ray, c.base_o)):
        p, valid = to_packets(recs, K, hit=not occluded)
        valid[:n] = np.where(np.random.RandomState(K).rand(n) < 0.7, -1, 0)
        dp, dv = _cuda(p), _cuda(valid)
        fn = c.lib.rtcb200OccludedNMDevice if occluded else c.lib.rtcb200IntersectNMDevice
        fn(C.c_void_p(dv.data_ptr()), c.sc, C.c_void_p(dp.data_ptr()), K, len(p), C.byref(c.lib.args()), _stream())
        torch.cuda.synchronize()
        c.lib.check(c.dev)
        got = from_packets(dp.cpu().numpy().view(packet_dtype(K, hit=not occluded)), n, hit=not occluded)
        active = valid[:n] == -1
        assert_same_records(got[active], base[active], f"K={K} occluded={occluded} active lanes")
        assert_same_records(got[~active], recs[~active], f"K={K} occluded={occluded} inactive lanes")


# ---- host-pointer pipeline -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d2h_partial", [0, 1])
@pytest.mark.parametrize("streams", [1, 6])
@pytest.mark.parametrize("scene", SCENES)
def test_host_pipeline(cases, scene, streams, d2h_partial):
    """rtcb200Intersect1M / Occluded1M / IntersectNM in chunks of 1024 rays (many chunks, a partial last one), over one or six
    streams, copying whole records back or (host_d2h_partial) only the bytes a query can change."""
    c = cases(scene)
    with tuning(c.lib, host_chunk_log2=10, host_streams=streams, host_d2h_partial=d2h_partial):
        got_i = c.lib.intersect(c.sc, host_copy(c.rh), "1M")
        got_o = c.lib.occluded(c.sc, host_copy(c.ray), "1M")
        got_p = c.lib.intersect(c.sc, host_copy(c.rh), "8M")
    c.lib.check(c.dev)
    assert_same_records(got_i, c.base_i, "rtcb200Intersect1M")
    assert_same_records(got_o, c.base_o, "rtcb200Occluded1M")
    assert_same_records(got_p, c.base_i, "rtcb200IntersectNM K=8")


# ---- fused hit gather ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("scene", SCENES)
def test_gather(cases, scene, mode):
    """rtcb200Intersect1MGatherDevice: the RTCRayHit records as the baseline and the compact {tfar, Ng, u, v, primID, geomID}
    records built from them (a miss: {tfar, 0, 0, 0, 0, 0, -1, -1}), in both delivery modes."""
    import torch
    from embree_b200 import sharding
    c = cases(scene)
    n = len(c.rh)
    with tuning(c.lib, gather_mode=mode):
        B = _cuda(c.rh)
        out = torch.full((n, 8), 7.0, device=B.device)
        c.lib.rtcb200Intersect1MGatherDevice(c.sc, C.c_void_p(B.data_ptr()), n, C.byref(c.lib.args()), _stream(), C.c_void_p(out.data_ptr()))
        torch.cuda.synchronize()
    c.lib.check(c.dev)
    assert_same_records(B.cpu().numpy().view(RAYHIT_DTYPE), c.base_i, "RTCRayHit records")
    want = sharding.compact_hits(torch.from_numpy(c.base_i.view(np.float32).reshape(-1, 24).copy()))
    miss = want.view(torch.int32)[:, 7] == -1
    want[miss, 1:6] = 0.0
    want.view(torch.int32)[miss, 6] = -1
    assert torch.equal(out.cpu().view(torch.int32), want.view(torch.int32))


# ---- counting kernels ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scene", SCENES)
def test_counting_kernels(cases, scene):
    """The STATS instantiations (rtcb200SetSceneStatCounters) write the same records and count every ray."""
    c = cases(scene)
    c.lib.rtcb200SetSceneStatCounters(c.sc, 1)
    try:
        c.lib.rtcb200ResetSceneStatCounters(c.sc)
        got_i = trace_device(c.lib, c.dev, c.sc, c.rh)
        st = c.lib.scene_stats(c.sc)
        got_o = trace_device(c.lib, c.dev, c.sc, c.ray, occluded=True)
    finally:
        c.lib.rtcb200SetSceneStatCounters(c.sc, 0)
    assert_same_records(got_i, c.base_i, "intersect")
    assert_same_records(got_o, c.base_o, "occluded")
    assert st.trav_rays == len(c.rh) and st.trav_nodes > st.trav_rays and st.trav_tris > 0, (st.trav_rays, st.trav_nodes, st.trav_tris)


def test_dense_leaves_overflow_the_queue(cases):
    """The terrain's leaf nodes carry enough triangle bits that the SPREAD queue must overflow: with tri_batch_min 32 a triangle
    step waits until all 32 lanes hold triangles, and a lane holds every triangle of the leaf slots its ray enters.  Most slots
    hold two or more triangles and a node's slots hold eight or more together, so 32 pending lanes bring far more than 32 items."""
    c = cases("terrain")
    N = bvh_check.Nodes(c.lib.scene_arrays(c.sc)["nodes"])
    bits = np.bitwise_count(np.bitwise_or.reduce(N.leaf, axis=1))            # triangle bits per node
    per_slot = np.bitwise_count(N.leaf[~N.inner & (N.leaf != 0)])
    assert np.median(bits[bits > 0]) >= 8 and (per_slot >= 2).mean() >= 0.6, (np.median(bits[bits > 0]), (per_slot >= 2).mean())
    cam = (c.rh["tnear"] == 0) & (c.rh["id"] >= 20011) & (c.rh["id"] < 20011 + 256 * 192)
    assert cam.sum() == 256 * 192 and (c.base_i["geomID"][cam] == 0).mean() > 0.4   # the lower part of the image sees the terrain


# ---- SPREAD off --------------------------------------------------------------------------------------------------------------
def test_tri_spread_matches_per_lane_kernel(b200):
    """The warp-wide triangle step (SPREAD, the shipped closest-hit kernel of triangle scenes) and the per-lane test ("tri_spread"
    0) accept by different rules -- SPREAD tests against the ray's own tfar and keeps t <= the hit so far, the per-lane test
    against the hit so far -- so they agree on the hit, not on every byte: ids identical except equal-distance ties, t / u / v / Ng
    bit-equal for the same primitive."""
    import torch
    lib, dev = b200
    v, t = scenes.triangle_sphere(300)
    sc, keep = build_scene(lib, dev, [(v, t, 0, 0xFFFFFFFF)])
    prim = scenes.primary_rays(640, 360, eye=(0.15, -0.1, 0.05), look=(0.3, 0.2, 1.0), device=torch.device("cuda", 0))
    a = lib.args()
    st = torch.cuda.current_stream().cuda_stream
    lib.rtcb200Intersect1MDevice(sc, C.c_void_p(prim.data_ptr()), prim.shape[0], C.byref(a), C.c_void_p(st))
    rays = scenes.diffuse_bounce_rays(prim, seed=1, replicate=8)
    out = []
    for spread in (0, 1):
        with tuning(lib, tri_spread=spread):
            B = rays.clone()
            lib.rtcb200Intersect1MDevice(sc, C.c_void_p(B.data_ptr()), B.shape[0], C.byref(a), C.c_void_p(st))
            torch.cuda.synchronize()
            lib.check(dev)
            out.append(scenes.as_numpy_rayhits(B.cpu()))
    rep = compare_hits(out[0], out[1], 1e-6)
    assert rep["hits"] > 1000000 and rep["id_mismatch"] == 0 and rep["hit_miss_disagree"] == 0 and rep["tie"] <= 50, rep
    same = (out[0]["primID"] == out[1]["primID"]) & (out[0]["geomID"] != 0xFFFFFFFF)
    for f in ("tfar", "u", "v", "Ng_x", "Ng_y", "Ng_z"):
        assert (out[0][f].view(np.uint32) == out[1][f].view(np.uint32))[same].all(), f
    lib.rtcReleaseScene(sc)


def test_filter_kernel_matches_per_lane_kernel(cases):
    """The filter-callback passes (an accept-all argument filter through rtcb200Intersect1M) run the FILTER instantiation, whose
    triangle test is the per-lane rule: with every candidate accepted its records equal "tri_spread" 0's byte for byte."""
    c = cases("sphere")
    rh = host_copy(c.rh[:40001])
    calls = [0]

    def accept(args):
        calls[0] += 1
    cb = FILTER_FUNCTION(accept)
    got = c.lib.intersect(c.sc, host_copy(rh), "1M", args=c.lib.args(filter=cb, invoke_argument_filter=True))
    c.lib.check(c.dev)
    with tuning(c.lib, tri_spread=0):
        want = trace_device(c.lib, c.dev, c.sc, rh)
    hits = (want["geomID"] != 0xFFFFFFFF).sum()
    assert calls[0] == hits > 1000, (calls[0], hits)
    assert_same_records(got, want, "accept-all filter against tri_spread 0")


# ---- the signed-zero stream --------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def zero_grid(b200):
    lib, dev = b200
    v, t, rays = signed_zero_grid()
    sc, keep = build_scene(lib, dev, [(v, t, 0, 0xFFFFFFFF)])
    base_i = trace_device(lib, dev, sc, rays)
    base_o = trace_device(lib, dev, sc, rays_of(rays), occluded=True)
    yield lib, dev, sc, v, t, rays, base_i, base_o
    lib.rtcReleaseScene(sc)


def test_signed_zero_hits_against_float64(zero_grid):
    """Every ray with tnear < 0 starts on the grid: it reports t = +0 or -0, on a triangle whose closed float64 triangle contains its
    origin.  A ray with tnear = 0 reports no zero-distance hit (the plane is all there is, so it misses)."""
    lib, dev, sc, v, t, rays, base_i, base_o = zero_grid
    cand = zero_distance_candidates(v, t, rays)
    neg = rays["tnear"] < 0
    assert cand.any(1).all()
    hit = base_i["geomID"] == 0
    assert hit[neg].all() and not hit[~neg].any()
    assert ((base_i["tfar"][neg].view(np.uint32) & 0x7FFFFFFF) == 0).all()
    k = np.nonzero(neg)[0]
    assert cand[k, base_i["primID"][k]].all()
    assert ((base_o["tfar"] == -np.inf) == neg).all()
    signs = base_i["tfar"][neg].view(np.uint32) >> 31
    assert signs.any() and not signs.all()          # both zeros are reported


@pytest.mark.parametrize("path", ["tri_step_32_1000", "permuted", "packets16", "host"])
def test_signed_zero_paths_agree(zero_grid, path):
    """Among candidates at equal distance the later one wins, -0 and +0 being equal: every path returns the baseline's records."""
    import torch
    lib, dev, sc, v, t, rays, base_i, base_o = zero_grid
    n = len(rays)
    ray = rays_of(rays)
    if path == "tri_step_32_1000":
        with tuning(lib, tri_batch_min=32, tri_wait_max=1000):
            got_i, got_o = trace_device(lib, dev, sc, rays), trace_device(lib, dev, sc, ray, occluded=True)
    elif path == "permuted":
        perm = np.random.RandomState(4).permutation(n)
        got_i, got_o = aligned_empty(n, RAYHIT_DTYPE), aligned_empty(n, RAY_DTYPE)
        got_i[perm] = trace_device(lib, dev, sc, host_copy(rays[perm]))
        got_o[perm] = trace_device(lib, dev, sc, host_copy(ray[perm]), occluded=True)
    elif path == "packets16":
        out = []
        for occluded, recs in ((False, rays), (True, ray)):
            p, valid = to_packets(recs, 16, hit=not occluded)
            dp, dv = _cuda(p), _cuda(valid)
            fn = lib.rtcb200OccludedNMDevice if occluded else lib.rtcb200IntersectNMDevice
            fn(C.c_void_p(dv.data_ptr()), sc, C.c_void_p(dp.data_ptr()), 16, len(p), C.byref(lib.args()), _stream())
            torch.cuda.synchronize()
            out.append(from_packets(dp.cpu().numpy().view(packet_dtype(16, hit=not occluded)), n, hit=not occluded))
        got_i, got_o = out
    else:
        got_i, got_o = lib.intersect(sc, host_copy(rays), "1M"), lib.occluded(sc, ray, "1M")
    lib.check(dev)
    assert_same_records(got_i, base_i, path + " intersect")
    assert_same_records(got_o, base_o, path + " occluded")


# ---- last: the tuning is back at the shipped values --------------------------------------------------------------------------
def test_zz_shipped_tuning_is_restored(cases):
    """After every test above, the first scene traced with no knob set writes the baseline's bytes again."""
    c = cases(SCENES[0])
    assert_same_records(trace_device(c.lib, c.dev, c.sc, c.rh), c.base_i, "intersect")
    assert_same_records(trace_device(c.lib, c.dev, c.sc, c.ray, occluded=True), c.base_o, "occluded")
