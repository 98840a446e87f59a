"""Ray queries from the caller's own CUDA kernels: include/embree4_b200_device.cuh and rtcb200GetSceneDeviceTraversable.

CPU: a user translation unit that includes only the public headers compiles for sm_90a with -I include, and two of them
device-link with -rdc=true.  GPU: tests/device_api/devtrace.cu traces from device code and every byte of every record (misses
included) must equal what rtcb200Intersect1MDevice / rtcb200Occluded1MDevice write for a copy of the same input, over triangle,
quad, instanced, curve, point, two-level, refitted and empty scenes, and for rays whose candidates tie at t = +0 / -0; plus the
getter's refusals."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from embree_b200 import scenes
from embree_b200.rtc import (FILTER_FUNCTION, RAY_DTYPE, RAYHIT_DTYPE, RTC_BUFFER_TYPE_VERTEX, DeviceTraversable, RayQueryContext,
                             _IntersectArguments, make_rayhits, rays_of)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDE = os.path.join(ROOT, "include")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
DEVTRACE = os.path.join(ROOT, "tests", "device_api", "_build", "libdevtrace.so")
N_RAYS = (1 << 20) + 5   # about 1 Mi rays, not a multiple of 32

USER_TU = r"""
#include "embree4_b200.h"
#include "embree4_b200_device.cuh"
__global__ void KERNEL(RTCB200DeviceTraversable t, RTCRayHit* rh, RTCRay* r, const RTCIntersectArguments* ia, const RTCOccludedArguments* oa, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  rtcb200TraversableIntersect1(t, rh + i, ia);
  rtcb200TraversableOccluded1(t, r + i);
  rtcb200TraversableOccluded1(t, r + i, oa);
}
void LAUNCH(RTCB200DeviceTraversable t, RTCRayHit* rh, RTCRay* r, int n) { KERNEL<<<(n + 127) / 128, 128>>>(t, rh, r, nullptr, nullptr, n); }
"""


def _user_tu(d, name):
    path = os.path.join(d, name + ".cu")
    with open(path, "w") as f:
        f.write(USER_TU.replace("KERNEL", name + "_kernel").replace("LAUNCH", name + "_launch"))
    return path


def _nvcc(args, cwd):
    r = subprocess.run([NVCC] + args, cwd=cwd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
    return r.stdout


def test_user_translation_unit_compiles_with_the_public_headers_only():
    with tempfile.TemporaryDirectory() as d:
        src = _user_tu(d, "user")
        _nvcc(["-std=c++17", *ARCH, "-I", INCLUDE, "-c", src, "-o", "user.o"], d)
        assert os.path.getsize(os.path.join(d, "user.o")) > 0


def test_two_translation_units_device_link_without_duplicate_symbols():
    with tempfile.TemporaryDirectory() as d:
        for name in ("a", "b"):
            _nvcc(["-std=c++17", *ARCH, "-rdc=true", "-Xcompiler", "-fPIC", "-I", INCLUDE, "-c", _user_tu(d, name), "-o", name + ".o"], d)
        _nvcc([*ARCH, "-dlink", "a.o", "b.o", "-o", "dlink.o", "-Xcompiler", "-fPIC"], d)
        _nvcc([*ARCH, "-rdc=true", "-shared", "-Xcompiler", "-fPIC", "a.o", "b.o", "-o", "libab.so"], d)
        assert os.path.getsize(os.path.join(d, "libab.so")) > 0


# ---- GPU -----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def devtrace():
    if not os.path.exists(DEVTRACE):
        subprocess.check_call([os.path.join(ROOT, "tests", "device_api", "build.sh")])
    L = C.CDLL(DEVTRACE)
    P = C.c_void_p
    L.devtrace_intersect.argtypes = [P, P, C.c_size_t, P, P]
    L.devtrace_occluded.argtypes = [P, P, C.c_size_t, P, P]
    L.devtrace_two_query.argtypes = [P, P, P, P, C.c_size_t, C.c_uint, C.c_float, P]
    L.devtrace_mixed.argtypes = [P, P, C.c_size_t, P]
    return L


def query_rays(n, center, radius, seed=1):
    """Incoherent rays from a sphere of `radius` around `center` towards random points inside it, with every case the API
    distinguishes: random geometry / instance masks, tnear > 0 with finite tfar, tfar < 0, and zero direction components."""
    rng = np.random.RandomState(seed)
    c = np.asarray(center, np.float32)
    o = rng.normal(size=(n, 3))
    o = o / np.linalg.norm(o, axis=1, keepdims=True) * radius + c
    inside = rng.uniform(-0.6, 0.6, (n, 3)) * radius + c
    d = (inside - o).astype(np.float32)
    o = o.astype(np.float32)
    q = n // 8
    d[q:2 * q, 0] = 0.0                       # zero direction components
    d[2 * q:3 * q, 1:] = 0.0
    o[2 * q:3 * q, 1:] = inside[2 * q:3 * q, 1:]   # (axis-parallel rays through the scene)
    r = make_rayhits(o, d)
    r["mask"][3 * q:4 * q] = rng.choice(np.array([0, 1, 2, 4, 5, 6, 0xFFFFFFFE, 0xFFFFFFFF], np.uint32), q)
    r["tnear"][4 * q:5 * q] = rng.uniform(0.0, 0.7, q).astype(np.float32)
    r["tfar"][4 * q:5 * q] = rng.uniform(0.6, 1.2, q).astype(np.float32)
    r["tfar"][5 * q:5 * q + q // 4] = -1.0      # tfar < 0
    r["tfar"][5 * q + q // 4:5 * q + q // 2] = -0.0
    return r


def _dev(a):
    import torch
    d = torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).cuda()
    torch.cuda.synchronize()   # the queries run on other streams
    return d


def _device_args(ctx):
    """RTCIntersectArguments (== RTCOccludedArguments' layout) followed by its RTCRayQueryContext, in device memory."""
    import torch
    buf = torch.zeros(48, dtype=torch.uint8, device="cuda")
    a = _IntersectArguments()
    a.flags, a.feature_mask, a.context, a.filter, a.intersect = 0, 0xFFFFFFFF, buf.data_ptr() + 32, None, None
    host = bytes(a) + bytes(ctx) + bytes(8)
    buf.copy_(torch.frombuffer(bytearray(host), dtype=torch.uint8))
    return buf


def compare_queries(lib, dev, devtrace, scene, rh, ctx=None, expect_hits=True):
    """Trace `rh` through the device functions and through the batched Device entry points (intersect and occluded, each on
    its own copy, on one stream) and require byte-identical records."""
    import torch
    t = lib.scene_device_traversable(scene)
    lib.check(dev)
    st = torch.cuda.Stream()
    host_args = lib.args(context=ctx) if ctx is not None else None
    dargs = _device_args(ctx) if ctx is not None else None
    dptr = C.c_void_p(dargs.data_ptr()) if dargs is not None else None
    r = rays_of(rh)
    a_i, b_i, a_o, b_o = _dev(rh), _dev(rh), _dev(r), _dev(r)
    with torch.cuda.stream(st):
        s = C.c_void_p(st.cuda_stream)
        assert devtrace.devtrace_intersect(C.byref(t), C.c_void_p(a_i.data_ptr()), len(rh), dptr, s) == 0
        lib.rtcb200Intersect1MDevice(scene, C.c_void_p(b_i.data_ptr()), len(rh), C.byref(host_args) if host_args else None, s)
        assert devtrace.devtrace_occluded(C.byref(t), C.c_void_p(a_o.data_ptr()), len(r), dptr, s) == 0
        lib.rtcb200Occluded1MDevice(scene, C.c_void_p(b_o.data_ptr()), len(r), C.byref(host_args) if host_args else None, s)
    st.synchronize()
    lib.check(dev)
    got_i, want_i = a_i.cpu().numpy().view(RAYHIT_DTYPE), b_i.cpu().numpy().view(RAYHIT_DTYPE)
    got_o, want_o = a_o.cpu().numpy().view(RAY_DTYPE), b_o.cpu().numpy().view(RAY_DTYPE)
    bad = np.nonzero((got_i.view(np.uint8).reshape(-1, 96) != want_i.view(np.uint8).reshape(-1, 96)).any(1))[0]
    assert len(bad) == 0, (len(bad), got_i[bad[:3]], want_i[bad[:3]])
    bad = np.nonzero((got_o.view(np.uint8).reshape(-1, 48) != want_o.view(np.uint8).reshape(-1, 48)).any(1))[0]
    assert len(bad) == 0, (len(bad), got_o[bad[:3]], want_o[bad[:3]])
    hits = want_i["geomID"] != 0xFFFFFFFF
    if expect_hits:
        assert hits.sum() > len(rh) // 20 and (~hits).sum() > 0, hits.sum()
        assert (want_o["tfar"] == -np.inf).sum() > 0
    return want_i


def _release(lib, *scs):
    for s in scs:
        lib.rtcReleaseScene(s)


@pytest.mark.gpu
@pytest.mark.parametrize("robust", [False, True])
@pytest.mark.parametrize("quality", [0, 1])
def test_triangle_sphere(b200, devtrace, quality, robust):
    lib, dev = b200
    sc = lib.rtcNewScene(dev)
    lib.rtcSetSceneFlags(sc, 4 if robust else 0)
    lib.rtcSetSceneBuildQuality(sc, quality)
    v, t = scenes.triangle_sphere(400)
    v2, t2 = scenes.triangle_sphere(60, center=(0.3, 0.2, -0.1), radius=0.4)
    _, k1 = lib.add_triangle_mesh(dev, sc, v, t, mask=1)
    _, k2 = lib.add_triangle_mesh(dev, sc, v2, t2, mask=2)
    lib.rtcCommitScene(sc)
    lib.check(dev)
    assert lib.scene_device_traversable(sc).general == 0
    out = compare_queries(lib, dev, devtrace, sc, query_rays(N_RAYS, (0, 0, 0), 2.0))
    assert set(np.unique(out["geomID"]).tolist()) == {0, 1, 0xFFFFFFFF}
    _release(lib, sc)


def _quad_instance_scene(lib, dev, robust):
    keep = []
    child = lib.rtcNewScene(dev)
    lib.rtcSetSceneFlags(child, 4 if robust else 0)
    v, q = scenes.quad_terrain(96)
    keep.append(lib.add_quad_mesh(dev, child, v, q, mask=0xFFFFFFFF)[1])
    lib.rtcCommitScene(child)
    top = lib.rtcNewScene(dev)
    lib.rtcSetSceneFlags(top, 4 if robust else 0)
    v2, q2 = scenes.quad_terrain(64, seed=3)
    keep.append(lib.add_quad_mesh(dev, top, v2 * np.float32(1.5) - np.float32([0, 0.8, 0]), q2, mask=0xFFFFFFFF)[1])
    rng = np.random.RandomState(2)
    for i in range(6):
        m, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        p = rng.uniform(-1.5, 1.5, 3)
        lib.add_instance(dev, top, child, np.concatenate([m[:, 0], m[:, 1], m[:, 2], p]).astype(np.float32), mask=[1, 2, 4, 3, 6, 0xFFFFFFFF][i])
    lib.rtcCommitScene(top)
    lib.check(dev)
    return top, child, keep


@pytest.mark.gpu
@pytest.mark.parametrize("robust", [False, True])
def test_quads_under_instances_with_seeded_instance_ids(b200, devtrace, robust):
    lib, dev = b200
    top, child, keep = _quad_instance_scene(lib, dev, robust)
    assert lib.scene_device_traversable(top).general == 1
    rh = query_rays(N_RAYS, (0, 0, 0), 4.0, seed=3)
    out = compare_queries(lib, dev, devtrace, top, rh)
    inst = out["instID"][out["geomID"] != 0xFFFFFFFF]
    assert (inst != 0xFFFFFFFF).any() and (inst == 0xFFFFFFFF).any()
    ctx = RayQueryContext(77, 99)   # args->context seeds the ids of hits that no instance sets
    out = compare_queries(lib, dev, devtrace, top, rh, ctx=ctx)
    direct = (out["geomID"] != 0xFFFFFFFF) & (out["instID"] == 77)
    assert direct.any() and (out["instPrimID"][direct] == 99).all()
    assert ((out["instID"] < 7) & (out["instPrimID"] == 0)).any()
    _release(lib, top, child)


@pytest.mark.gpu
def test_scene_of_every_kind_with_instances(b200, devtrace):
    from tests.test_interpolate import mixed_scene
    lib, dev = b200
    top, child, keep = mixed_scene(lib, dev)
    assert lib.scene_device_traversable(top).curves == 2
    out = compare_queries(lib, dev, devtrace, top, query_rays(N_RAYS, (0, 0, 0), 8.0, seed=5))
    hit = out["geomID"] != 0xFFFFFFFF
    assert len(set(zip(out["instID"][hit].tolist(), out["geomID"][hit].tolist()))) >= 20
    _release(lib, top, child)


@pytest.mark.gpu
def test_points_only_scene(b200, devtrace):
    lib, dev = b200
    rng = np.random.RandomState(6)
    sc = lib.rtcNewScene(dev)
    keep = []
    for k, kind in enumerate(("sphere", "disc", "oriented_disc")):
        pv = np.concatenate([rng.normal(size=(20000, 3)), rng.uniform(0.005, 0.03, (20000, 1))], 1).astype(np.float32)
        nrm = rng.normal(size=(20000, 3)).astype(np.float32)
        keep.append(lib.add_points(dev, sc, pv, kind, normals=nrm if kind == "oriented_disc" else None, mask=1 << k)[1])
    lib.rtcCommitScene(sc)
    lib.check(dev)
    assert lib.scene_device_traversable(sc).curves == 1
    compare_queries(lib, dev, devtrace, sc, query_rays(N_RAYS, (0, 0, 0), 3.0, seed=7))
    _release(lib, sc)


@pytest.mark.gpu
def test_two_level_and_refitted_dynamic_scenes(b200, devtrace):
    from tests.test_gpu_parity import _dynamic_meshes
    lib, dev = b200
    meshes = _dynamic_meshes(24)
    sc = lib.rtcNewScene(dev)
    lib.rtcSetSceneFlags(sc, 1)   # DYNAMIC
    bufs = [lib.add_triangle_mesh(dev, sc, v, t, mask=0xFFFFFFFF) for v, t in meshes]
    lib.rtcCommitScene(sc)
    rh = query_rays(N_RAYS, (0, 0, 0), 5.0, seed=8)
    vpad = bufs[2][1][0]
    vpad[:len(meshes[2][0]) * 3] += np.float32(0.35)   # one mesh moves: the commit re-assembles the kept per-mesh BVHs
    g = lib.rtcGetGeometry(sc, 2)
    lib.rtcUpdateGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0)
    lib.rtcCommitGeometry(g)
    lib.rtcCommitScene(sc)
    lib.check(dev)
    assert lib.scene_stats(sc).builder == 3
    compare_queries(lib, dev, devtrace, sc, rh)   # a fresh traversable after the re-commit
    _release(lib, sc)

    v, t = scenes.triangle_sphere(200)
    sc = lib.rtcNewScene(dev)
    lib.rtcSetSceneFlags(sc, 1)
    _, (vpad, _i) = lib.add_triangle_mesh(dev, sc, v, t, mask=0xFFFFFFFF, quality=3)   # RTC_BUILD_QUALITY_REFIT
    lib.rtcCommitScene(sc)
    vpad[:v.size] = (v * np.float32([1.3, 1.0, 0.8])).ravel()
    g = lib.rtcGetGeometry(sc, 0)
    lib.rtcUpdateGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0)
    lib.rtcCommitGeometry(g)
    lib.rtcCommitScene(sc)
    lib.check(dev)
    assert lib.scene_stats(sc).builder == 2
    compare_queries(lib, dev, devtrace, sc, query_rays(N_RAYS, (0, 0, 0), 2.5, seed=9))
    _release(lib, sc)


@pytest.mark.gpu
def test_signed_zero_distance_ties(b200, devtrace):
    """Origins exactly on a planar grid with tnear < 0: each ray meets several candidates at t = +0 or -0, and the device query
    must pick the same winner as the batched kernels' warp-wide triangle step (the later candidate, the two zeros being equal)."""
    from tests.parity import signed_zero_grid
    lib, dev = b200
    v, t, rh = signed_zero_grid()
    sc = lib.rtcNewScene(dev)
    _, keep = lib.add_triangle_mesh(dev, sc, v, t, mask=0xFFFFFFFF)
    lib.rtcCommitScene(sc)
    lib.check(dev)
    out = compare_queries(lib, dev, devtrace, sc, rh)
    neg = rh["tnear"] < 0
    assert (out["geomID"][neg] == 0).all() and ((out["tfar"][neg].view(np.uint32) & 0x7FFFFFFF) == 0).all()
    _release(lib, sc)


@pytest.mark.gpu
def test_empty_scene_leaves_every_record_untouched(b200, devtrace):
    lib, dev = b200
    sc = lib.rtcNewScene(dev)
    lib.rtcCommitScene(sc)
    lib.check(dev)
    t = lib.scene_device_traversable(sc)
    lib.check(dev)
    assert t.root_valid == 0
    rh = query_rays(N_RAYS, (0, 0, 0), 1.0)
    out = compare_queries(lib, dev, devtrace, sc, rh, expect_hits=False)
    assert out.tobytes() == rh.tobytes()
    _release(lib, sc)


@pytest.mark.gpu
def test_two_queries_per_thread_and_mixed_warps(b200, devtrace):
    """Launcher (b): each thread traces its ray, forms and writes a secondary ray at the hit and traces it too -- both results
    equal the batched call on the same rays.  Launcher (c): even lanes intersect, odd lanes test occlusion, in one warp."""
    import torch
    from tests.test_interpolate import mixed_scene
    lib, dev = b200
    top, child, keep = mixed_scene(lib, dev)
    t = lib.scene_device_traversable(top)
    lib.check(dev)
    rh = query_rays(N_RAYS, (0, 0, 0), 8.0, seed=11)
    st = torch.cuda.Stream()
    a, sec_in, sec_out = _dev(rh), torch.zeros_like(_dev(rh)), torch.zeros_like(_dev(rh))
    primary, mixed = _dev(rh), _dev(rh)
    with torch.cuda.stream(st):
        s = C.c_void_p(st.cuda_stream)
        assert devtrace.devtrace_two_query(C.byref(t), C.c_void_p(a.data_ptr()), C.c_void_p(sec_in.data_ptr()), C.c_void_p(sec_out.data_ptr()),
                                           len(rh), 1234, 1e-3, s) == 0
        assert devtrace.devtrace_mixed(C.byref(t), C.c_void_p(mixed.data_ptr()), len(rh), s) == 0
        lib.rtcb200Intersect1MDevice(top, C.c_void_p(primary.data_ptr()), len(rh), None, s)
        secondary = sec_in.clone()
        lib.rtcb200Intersect1MDevice(top, C.c_void_p(secondary.data_ptr()), len(rh), None, s)
    st.synchronize()
    lib.check(dev)
    assert torch.equal(a, primary)
    sec = secondary.cpu().numpy().view(RAYHIT_DTYPE)
    got = sec_out.cpu().numpy().view(RAYHIT_DTYPE)
    bad = np.nonzero((got.view(np.uint8).reshape(-1, 96) != sec.view(np.uint8).reshape(-1, 96)).any(1))[0]
    assert len(bad) == 0, (len(bad), sec_in.cpu().numpy().view(RAYHIT_DTYPE)[bad[:4]], got[bad[:4]], sec[bad[:4]])
    assert (sec["geomID"] != 0xFFFFFFFF).sum() > len(rh) // 20
    # (c): even records as the batched intersect, odd ones as the batched occluded on their RTCRay halves
    want_o = _dev(rays_of(rh))
    with torch.cuda.stream(st):
        lib.rtcb200Occluded1MDevice(top, C.c_void_p(want_o.data_ptr()), len(rh), None, C.c_void_p(st.cuda_stream))
    st.synchronize()
    got = mixed.cpu().numpy().view(np.uint8).reshape(-1, 96)
    want_i = primary.cpu().numpy().view(np.uint8).reshape(-1, 96)
    assert (got[0::2] == want_i[0::2]).all()
    assert (got[1::2, :48] == want_o.cpu().numpy().reshape(-1, 48)[1::2]).all()
    assert (got[1::2, 48:] == rh.view(np.uint8).reshape(-1, 96)[1::2, 48:]).all()   # occluded leaves the hit half alone
    _release(lib, top, child)


# ---- getter refusals -------------------------------------------------------------------------------------------------------
def _refused(lib, dev, sc):
    t = DeviceTraversable()
    C.memset(C.byref(t), 0xAB, C.sizeof(t))
    lib.rtcb200GetSceneDeviceTraversable(sc, C.byref(t))
    err = lib.rtcGetDeviceError(dev)
    return err == 3 and bytes(t) == bytes(C.sizeof(t)), err


def _accepted(lib, dev, sc):
    t = lib.scene_device_traversable(sc)
    return lib.rtcGetDeviceError(dev) == 0 and t.root_valid == 1 and t.nodes and t.records


@pytest.mark.gpu
def test_getter_refusals(b200):
    lib, dev = b200
    v, t = scenes.triangle_sphere(20)
    keep = []
    sc = lib.rtcNewScene(dev)
    keep.append(lib.add_triangle_mesh(dev, sc, v, t)[1])
    assert _refused(lib, dev, sc)[0], "an uncommitted scene is refused"
    lib.rtcCommitScene(sc)
    assert _accepted(lib, dev, sc)

    cb = FILTER_FUNCTION(lambda args: None)
    g = lib.rtcGetGeometry(sc, 0)
    lib.rtcSetGeometryIntersectFilterFunction(g, C.cast(cb, C.c_void_p))
    assert _refused(lib, dev, sc)[0], "a geometry intersect filter is refused"
    lib.rtcSetGeometryIntersectFilterFunction(g, None)
    assert _accepted(lib, dev, sc)
    lib.rtcSetGeometryEnableFilterFunctionFromArguments(g, True)   # argument filters never run on the device: accepted
    assert _accepted(lib, dev, sc)
    lib.rtcSetGeometryEnableFilterFunctionFromArguments(g, False)

    top = lib.rtcNewScene(dev)
    lib.add_instance(dev, top, sc, np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0.5, 0, 0], np.float32))
    lib.rtcCommitScene(top)
    assert _accepted(lib, dev, top)
    lib.rtcSetGeometryOccludedFilterFunction(g, C.cast(cb, C.c_void_p))
    assert _refused(lib, dev, top)[0], "an occluded filter on an instanced child is refused"
    assert _refused(lib, dev, sc)[0]
    lib.rtcSetGeometryOccludedFilterFunction(g, None)
    assert _accepted(lib, dev, top) and _accepted(lib, dev, sc)
    lib.check(dev)
    _release(lib, top, sc)
