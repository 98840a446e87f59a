"""Shading from the caller's own CUDA kernels: rtcb200GetGeometryUserDataFromTraversable, rtcb200GetGeometryTransformFromTraversable
and rtcb200Interpolate1 (include/embree4_b200_device.cuh) with rtcb200GetSceneDeviceInterpolator.

CPU: a user translation unit that calls all four compiles with -I include only and two of them device-link with -rdc=true; the C
structs match rtc.py; the shared transform permutation, instantiated on the host, writes the reference's storeTransform layout.
GPU (tests/device_shading/devshade.cu): per-hit interpolation equals rtcb200InterpolateHitsDevice byte for byte (misses untouched,
points NaN) over the scene of every kind with instances, a scene of wide attributes, two-level and refitted dynamic scenes; a kernel
that traces and interpolates equals the two batched calls; user data and transforms equal the host getters, with the snapshot
semantics; the interpolator getter's refusals."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from embree_b200 import rtc, scenes
from embree_b200.rtc import (INTERP_OUTPUTS, RAYHIT_DTYPE, RTC_BUFFER_TYPE_VERTEX, RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, RTC_FORMAT_FLOAT,
                             DeviceGeometryHeader, DeviceGeometryInfo, DeviceInterpolateArguments, DeviceInterpolator)
from tests.test_device_traversal import ARCH, INCLUDE, ROOT, _nvcc

DEVSHADE = os.path.join(ROOT, "tests", "device_shading", "_build", "libdevshade.so")
INVALID = 0xFFFFFFFF
SENTINEL = -7.5
FMT_ROW, FMT_COL, FMT_4X4 = 0x9134, 0x9234, 0x9244

USER_TU = r"""
#include "embree4_b200.h"
#include "embree4_b200_device.cuh"
__global__ void NAME_kernel(RTCB200DeviceTraversable t, RTCB200DeviceInterpolator ip, RTCRayHit* rh, float* out, void** ud, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  rtcb200TraversableIntersect1(t, rh + i);
  RTCB200DeviceInterpolateArguments a = {rh[i].hit.geomID, rh[i].hit.instID[0], rh[i].hit.primID, rh[i].hit.u, rh[i].hit.v, out + 16 * i};
  a.valueCount = 3;
  rtcb200Interpolate1(ip, &a);
  rtcb200GetGeometryTransformFromTraversable(t, rh[i].hit.instID[0], 0.0f, RTC_FORMAT_FLOAT3X4_ROW_MAJOR, out + 16 * i + 3);
  ud[i] = rtcb200GetGeometryUserDataFromTraversable(t, rh[i].hit.geomID);
}
void NAME_launch(RTCB200DeviceTraversable t, RTCB200DeviceInterpolator ip, RTCRayHit* rh, float* out, void** ud, int n) {
  NAME_kernel<<<(n + 127) / 128, 128>>>(t, ip, rh, out, ud, n);
}
"""


def _user_tu(d, name):
    path = os.path.join(d, name + ".cu")
    with open(path, "w") as f:
        f.write(USER_TU.replace("NAME", name))
    return path


def test_user_translation_unit_with_shading_calls_compiles_with_the_public_headers_only():
    with tempfile.TemporaryDirectory() as d:
        _nvcc(["-std=c++17", *ARCH, "-I", INCLUDE, "-c", _user_tu(d, "user"), "-o", "user.o"], d)
        assert os.path.getsize(os.path.join(d, "user.o")) > 0


def test_two_translation_units_with_shading_calls_device_link():
    with tempfile.TemporaryDirectory() as d:
        for name in ("a", "b"):
            _nvcc(["-std=c++17", *ARCH, "-rdc=true", "-Xcompiler", "-fPIC", "-I", INCLUDE, "-c", _user_tu(d, name), "-o", name + ".o"], d)
        _nvcc([*ARCH, "-rdc=true", "-shared", "-Xcompiler", "-fPIC", "a.o", "b.o", "-o", "libab.so"], d)
        assert os.path.getsize(os.path.join(d, "libab.so")) > 0


def test_struct_layouts_match_the_bindings():
    src = r"""
#include <stddef.h>
#include "embree4_b200.h"
_Static_assert(sizeof(struct RTCB200DeviceTraversable) == 48 && offsetof(struct RTCB200DeviceTraversable, geometries) == 40, "traversable");
_Static_assert(sizeof(struct RTCB200DeviceGeometry) == 16 && sizeof(struct RTCB200DeviceGeometryHeader) == 16, "entry, header");
_Static_assert(sizeof(struct RTCB200DeviceGeometryInfo) == 64 && offsetof(struct RTCB200DeviceGeometryInfo, xfm) == 12, "info");
_Static_assert(offsetof(struct RTCB200DeviceGeometryHeader, count) == 8, "count");
_Static_assert(sizeof(struct RTCB200DeviceInterpolator) == 16 && offsetof(struct RTCB200DeviceInterpolator, nentries) == 8, "interpolator");
_Static_assert(sizeof(struct RTCB200DeviceInterpolateArguments) == 80, "arguments");
_Static_assert(offsetof(struct RTCB200DeviceInterpolateArguments, v) == 16 && offsetof(struct RTCB200DeviceInterpolateArguments, P) == 24, "u v P");
_Static_assert(offsetof(struct RTCB200DeviceInterpolateArguments, ddPdudv) == 64, "ddPdudv");
_Static_assert(offsetof(struct RTCB200DeviceInterpolateArguments, valueCount) == 72, "valueCount");
"""
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "layout.c")
        with open(path, "w") as f:
            f.write(src)
        r = subprocess.run(["cc", "-std=c11", "-fsyntax-only", "-I", INCLUDE, path], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        assert r.returncode == 0, r.stdout
    assert C.sizeof(rtc.DeviceTraversable) == 48 and rtc.DeviceTraversable.geometries.offset == 40
    assert C.sizeof(DeviceGeometryHeader) == 16 and DeviceGeometryHeader.count.offset == 8
    assert C.sizeof(DeviceGeometryInfo) == 64 and DeviceGeometryInfo.xfm.offset == 12
    assert C.sizeof(DeviceInterpolator) == 16 and DeviceInterpolator.nentries.offset == 8
    assert C.sizeof(DeviceInterpolateArguments) == 80 and DeviceInterpolateArguments.P.offset == 24
    assert DeviceInterpolateArguments.ddPdudv.offset == 64 and DeviceInterpolateArguments.valueCount.offset == 72


def test_transform_permutation_writes_the_reference_layout():
    """transform_format.cuh compiled by the host compiler, on local2world columns vx = (1,2,3), vy = (4,5,6), vz = (7,8,9), p = (10,11,12):
    the layouts of the reference's storeTransform (kernels/common/rtcore.h:125-155), written out by hand."""
    src = r"""
#include <stdio.h>
#include "transform_format.cuh"
int main() {
  const float m[12] = {1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12};
  const unsigned f[4] = {0x9134, 0x9234, 0x9244, 0x9001};
  for (int k = 0; k < 4; ++k) {
    float x[16];
    for (int j = 0; j < 16; ++j) x[j] = -1.0f;
    const bool ok = rtk::store_transform(m, f[k], x);
    printf("%d", ok ? 1 : 0);
    for (int j = 0; j < 16; ++j) printf(" %g", x[j]);
    printf("\n");
  }
}
"""
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "tf.cpp")
        with open(path, "w") as f:
            f.write(src)
        exe = os.path.join(d, "tf")
        r = subprocess.run(["c++", "-std=c++17", "-I", os.path.join(ROOT, "embree_b200", "csrc"), path, "-o", exe],
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        assert r.returncode == 0, r.stdout
        rows = [[float(x) for x in line.split()] for line in subprocess.check_output([exe], text=True).splitlines()]
    row_major = [1, 4, 7, 10, 2, 5, 8, 11, 3, 6, 9, 12]
    col_major = [1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12]
    col_4x4 = [1, 2, 3, 0, 4, 5, 6, 0, 7, 8, 9, 0, 10, 11, 12, 1]
    assert rows[0] == [1] + row_major + [-1] * 4
    assert rows[1] == [1] + col_major + [-1] * 4
    assert rows[2] == [1] + col_4x4
    assert rows[3] == [0] + [-1] * 16                  # an unknown format writes nothing


# ---- GPU -----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def devshade():
    if not os.path.exists(DEVSHADE):
        subprocess.check_call([os.path.join(ROOT, "tests", "device_shading", "build.sh")])
    L = C.CDLL(DEVSHADE)
    P = C.c_void_p
    L.devshade_interpolate.argtypes = [P, C.c_int, P, C.c_size_t, C.c_uint, P, P]
    L.devshade_trace_interpolate.argtypes = [P, P, P, C.c_size_t, C.c_uint, P, P]
    L.devshade_user_data.argtypes = [P, P, C.c_size_t, P, P]
    L.devshade_transform.argtypes = [P, P, C.c_size_t, C.c_uint, P, P]
    return L


def _outs(M, vc, want=INTERP_OUTPUTS):
    import torch
    return {k: torch.full((M, vc), SENTINEL, dtype=torch.float32, device="cuda") for k in want}


def _ptrs(outs):
    return (C.c_void_p * 6)(*[outs[k].data_ptr() if k in outs else None for k in INTERP_OUTPUTS])


def device_interpolate(lib, dev, L, scene, d_hits, bt, slot, vc, stream):
    """rtcb200Interpolate1 of every record of d_hits (a CUDA tensor of RTCRayHit records) on `stream`: {output: [M, vc]}."""
    import torch
    ip =lib.scene_device_interpolator(scene, bt, slot)
    lib.check(dev)
    M = d_hits.numel() // 96
    o = _outs(M, vc)
    torch.cuda.synchronize()   # the fills run on the current stream, the kernel on `stream`
    assert L.devshade_interpolate(C.byref(ip), 0, C.c_void_p(d_hits.data_ptr()), M, vc, _ptrs(o), C.c_void_p(stream.cuda_stream)) == 0
    return o


def compare_with_batched(lib, dev, L, scene, d_hits, bt, slot, vc, expect_nan=True):
    """Per-hit and batched interpolation of the same hits on one stream, every output byte-identical (the device results
    transposed); misses keep the sentinel.  Returns the hit records and the per-hit results."""
    import torch
    st = torch.cuda.Stream()
    M = d_hits.numel() // 96
    want = {k: torch.full((vc, M), SENTINEL, dtype=torch.float32, device="cuda") for k in INTERP_OUTPUTS}
    got = device_interpolate(lib, dev, L, scene, d_hits, bt, slot, vc, st)   # synchronises before it launches
    lib.interpolate_hits(scene, d_hits, bt, slot, vc, want=INTERP_OUTPUTS, stream=st, out=want)
    st.synchronize()
    lib.check(dev)
    hits = d_hits.cpu().numpy().view(RAYHIT_DTYPE).reshape(-1)
    miss = hits["geomID"] == INVALID
    assert miss.any() and (~miss).sum() > M // 20
    for k in INTERP_OUTPUTS:
        g, w = got[k].cpu().numpy().T, want[k].cpu().numpy()
        assert g.view(np.uint32).tobytes() == w.view(np.uint32).tobytes(), (bt, slot, vc, k)
        assert (g[:, miss] == SENTINEL).all()
    nan = np.isnan(got["P"].cpu().numpy()).all(1)
    assert nan.any() == expect_nan and not (nan & miss).any()
    return hits, got


def _trace(lib, scene, rh):
    import torch
    d = torch.from_numpy(rh.view(np.uint8).copy()).cuda()
    st = torch.cuda.current_stream()
    lib.rtcb200Intersect1MDevice(scene, C.c_void_p(d.data_ptr()), len(rh), C.byref(lib.args()), C.c_void_p(st.cuda_stream))
    torch.cuda.synchronize()
    return d


@pytest.mark.gpu
def test_interpolation_equals_the_batched_call_on_the_scene_of_every_kind(b200, devshade):
    """Vertex buffers (FLOAT3 meshes, FLOAT4 curves), attribute slot 0 (FLOAT3 at a 20-byte stride: scalar loads) and slot 1 (FLOAT4
    at 16 bytes: 16-byte loads), through six instances; points give NaN."""
    from tests.test_interpolate import mixed_scene, rays
    lib, dev = b200
    top, child, keep = mixed_scene(lib, dev)
    d = _trace(lib, top, rays((1 << 20) + 3))
    for bt, slot, vc in ((RTC_BUFFER_TYPE_VERTEX, 0, 1), (RTC_BUFFER_TYPE_VERTEX, 0, 3), (RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 0, 3),
                         (RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 1, 1), (RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 1, 4)):
        hits, got = compare_with_batched(lib, dev, devshade, top, d, bt, slot, vc)
    hit = hits["geomID"] != INVALID
    assert (hits["instID"][hit] != INVALID).any() and (hits["instID"][hit] == INVALID).any()
    lib.rtcReleaseScene(top)
    lib.rtcReleaseScene(child)


def _wide_scene(lib, dev):
    """Triangles, quads, Bezier and linear curves with FLOAT16 attributes at a stride of 64 bytes (slot 0) and 68 bytes (slot 1)."""
    from tests.test_interpolate import add_geometry
    rng = np.random.RandomState(12)
    keep = []
    sc = lib.rtcNewScene(dev)

    def attrs(n):
        return [(rng.normal(size=(n, 16)).astype(np.float32), RTC_FORMAT_FLOAT + 15, 64), (rng.normal(size=(n, 17)).astype(np.float32), RTC_FORMAT_FLOAT + 15, 68)]
    v, t = scenes.triangle_sphere(60)
    v = np.concatenate([v, np.zeros((1, 3), np.float32)]).astype(np.float32)
    add_geometry(lib, dev, sc, 0, v, t, attrs=attrs(len(v)), keep=keep)
    gx, gy = np.meshgrid(np.linspace(-2, 2, 13), np.linspace(-2, 2, 13))
    qv = np.concatenate([np.stack([gx.ravel(), gy.ravel(), np.full(gx.size, -1.2)], 1), np.zeros((1, 3))]).astype(np.float32)
    a = np.arange(12 * 13).reshape(12, 13)[:, :12].ravel()
    qi = np.stack([a, a + 1, a + 14, a + 13], 1).astype(np.uint32)
    add_geometry(lib, dev, sc, 1, qv, qi, attrs=attrs(len(qv)), keep=keep)
    cv, ci, _ = scenes.cubic_hair(200, "bezier", knots=7, seed=3, radius=0.9, step=0.12, width=0.03)
    add_geometry(lib, dev, sc, 25, np.ascontiguousarray(cv, np.float32), np.ascontiguousarray(ci, np.uint32), attrs=attrs(len(cv)), keep=keep)
    lv, li, _ = scenes.hair_ball(300, 4, seed=4, radius=0.8, length=0.6, width=0.04)
    add_geometry(lib, dev, sc, 17, np.ascontiguousarray(lv, np.float32), np.ascontiguousarray(li, np.uint32), attrs=attrs(len(lv)), keep=keep)
    lib.rtcCommitScene(sc)
    lib.check(dev)
    return sc, keep


@pytest.mark.gpu
def test_interpolation_equals_the_batched_call_for_wide_attributes(b200, devshade):
    """valueCount 5 and 16 (the widest format) with 16-byte loads (stride 64) and scalar loads (stride 68)."""
    from tests.test_interpolate import rays
    lib, dev = b200
    sc, keep = _wide_scene(lib, dev)
    d = _trace(lib, sc, rays(1 << 18, seed=13, spread=2.0))
    for slot in (0, 1):
        for vc in (5, 16):
            compare_with_batched(lib, dev, devshade, sc, d, RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, slot, vc, expect_nan=False)
    lib.rtcReleaseScene(sc)


@pytest.mark.gpu
def test_interpolation_equals_the_batched_call_on_two_level_and_refitted_scenes(b200, devshade):
    from tests.test_device_traversal import query_rays
    from tests.test_gpu_parity import _dynamic_meshes
    lib, dev = b200
    meshes = _dynamic_meshes(24)
    sc = lib.rtcNewScene(dev)
    lib.rtcSetSceneFlags(sc, 1)
    bufs = [lib.add_triangle_mesh(dev, sc, v, t, mask=0xFFFFFFFF) for v, t in meshes]
    lib.rtcCommitScene(sc)
    first = lib.scene_device_interpolator(sc, RTC_BUFFER_TYPE_VERTEX, 0)
    bufs[2][1][0][:len(meshes[2][0]) * 3] += np.float32(0.35)
    g = lib.rtcGetGeometry(sc, 2)
    lib.rtcUpdateGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0)
    lib.rtcCommitGeometry(g)
    lib.rtcCommitScene(sc)
    lib.check(dev)
    assert lib.scene_stats(sc).builder == 3
    d = _trace(lib, sc, query_rays(1 << 20, (0, 0, 0), 5.0, seed=8))
    hits, _ = compare_with_batched(lib, dev, devshade, sc, d, RTC_BUFFER_TYPE_VERTEX, 0, 3, expect_nan=False)
    assert (hits["geomID"] == 2).sum() > 100
    again = lib.scene_device_interpolator(sc, RTC_BUFFER_TYPE_VERTEX, 0)
    assert again.table and again.nentries == 24 and first.nentries == 24
    lib.rtcReleaseScene(sc)

    v, t = scenes.triangle_sphere(200)
    sc = lib.rtcNewScene(dev)
    lib.rtcSetSceneFlags(sc, 1)
    _, (vpad, _i) = lib.add_triangle_mesh(dev, sc, v, t, mask=0xFFFFFFFF, quality=3)
    lib.rtcCommitScene(sc)
    vpad[:v.size] = (v * np.float32([1.3, 1.0, 0.8])).ravel()
    g = lib.rtcGetGeometry(sc, 0)
    lib.rtcUpdateGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0)
    lib.rtcCommitGeometry(g)
    lib.rtcCommitScene(sc)
    lib.check(dev)
    assert lib.scene_stats(sc).builder == 2
    d = _trace(lib, sc, query_rays(1 << 20, (0, 0, 0), 2.5, seed=9))
    compare_with_batched(lib, dev, devshade, sc, d, RTC_BUFFER_TYPE_VERTEX, 0, 3, expect_nan=False)
    lib.rtcReleaseScene(sc)


@pytest.mark.gpu
def test_trace_and_interpolate_in_one_thread_equals_the_batched_calls(b200, devshade):
    import torch
    from tests.test_interpolate import mixed_scene, rays
    lib, dev = b200
    top, child, keep = mixed_scene(lib, dev)
    rh = rays((1 << 20) + 3, seed=14)
    vc = 4
    t = lib.scene_device_traversable(top)
    ip = lib.scene_device_interpolator(top, RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 1)
    lib.check(dev)
    d = torch.from_numpy(rh.view(np.uint8).copy()).cuda()
    o = _outs(len(rh), vc)
    torch.cuda.synchronize()
    st = torch.cuda.Stream()
    assert devshade.devshade_trace_interpolate(C.byref(t), C.byref(ip), C.c_void_p(d.data_ptr()), len(rh), vc, _ptrs(o), C.c_void_p(st.cuda_stream)) == 0
    w = _trace(lib, top, rh)
    want = lib.interpolate_hits(top, w, RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 1, vc, want=INTERP_OUTPUTS,
                                out={k: torch.full((vc, len(rh)), SENTINEL, dtype=torch.float32, device="cuda") for k in INTERP_OUTPUTS})
    torch.cuda.synchronize()
    lib.check(dev)
    assert torch.equal(d, w)   # the records
    for k in INTERP_OUTPUTS:
        assert o[k].cpu().numpy().T.tobytes() == want[k].cpu().numpy().tobytes(), k
    lib.rtcReleaseScene(top)
    lib.rtcReleaseScene(child)


# ---- user data and transforms ----------------------------------------------------------------------------------------------
def _host(lib):
    f = lib.dll.rtcGetGeometryUserDataFromScene
    f.restype, f.argtypes = C.c_void_p, [C.c_void_p, C.c_uint]
    g = lib.dll.rtcGetGeometryTransformFromScene
    g.restype, g.argtypes = None, [C.c_void_p, C.c_uint, C.c_float, C.c_int, C.c_void_p]
    return f, g


def _device_user_data(lib, L, t, ids):
    import torch
    d_ids = torch.from_numpy(np.asarray(ids, np.uint32).view(np.int32)).cuda()
    out = torch.full((len(ids),), -1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    assert L.devshade_user_data(C.byref(t), C.c_void_p(d_ids.data_ptr()), len(ids), C.c_void_p(out.data_ptr()), None) == 0
    torch.cuda.synchronize()
    return out.cpu().numpy().view(np.uint64)


def _device_transform(lib, L, t, ids, fmt):
    import torch
    d_ids = torch.from_numpy(np.asarray(ids, np.uint32).view(np.int32)).cuda()
    out = torch.full((len(ids), 16), SENTINEL, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    assert L.devshade_transform(C.byref(t), C.c_void_p(d_ids.data_ptr()), len(ids), fmt, C.c_void_p(out.data_ptr()), None) == 0
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _every_kind_with_holes(lib, dev):
    """geomIDs 0..7: triangles, quads, a Bezier curve set, sphere points, two instances, a disabled mesh, and a detached slot (5)."""
    from tests.test_interpolate import add_geometry
    keep = []
    child = lib.rtcNewScene(dev)
    v, t = scenes.triangle_sphere(10)
    keep.append(lib.add_triangle_mesh(dev, child, v, t)[1])
    lib.rtcCommitScene(child)
    sc = lib.rtcNewScene(dev)
    keep.append(lib.add_triangle_mesh(dev, sc, v, t)[1])                                            # 0
    qv = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0], [0, 0, 0]], np.float32)
    add_geometry(lib, dev, sc, 1, qv, np.array([[0, 1, 2, 3]], np.uint32), keep=keep)                 # 1
    cv, ci, _ = scenes.cubic_hair(10, "bezier", knots=7, seed=1)
    add_geometry(lib, dev, sc, 25, np.ascontiguousarray(cv, np.float32), np.ascontiguousarray(ci, np.uint32), keep=keep)   # 2
    keep.append(lib.add_points(dev, sc, np.array([[0, 0, 3, 0.1], [1, 0, 3, 0.1]], np.float32))[1])  # 3
    lib.add_instance(dev, sc, child, np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 2, 0, 0], np.float32))    # 4
    keep.append(lib.add_triangle_mesh(dev, sc, v, t)[1])                                            # 5, detached below
    lib.add_instance(dev, sc, child, np.array([0, 2, 0, -1, 0, 0, 0, 0, 0.5, 1, 2, 3], np.float32))  # 6
    keep.append(lib.add_triangle_mesh(dev, sc, v, t)[1])                                            # 7, disabled
    lib.rtcDisableGeometry(lib.rtcGetGeometry(sc, 7))
    lib.rtcDetachGeometry(sc, 5)
    for gid in (0, 1, 2, 3, 4, 6, 7):
        lib.rtcSetGeometryUserData(lib.rtcGetGeometry(sc, gid), 0x1000 * (gid + 1) + 8)
    lib.rtcSetGeometryUserData(lib.rtcGetGeometry(child, 0), 0x77000)
    lib.rtcCommitScene(sc)
    lib.check(dev)
    return sc, child, keep


@pytest.mark.gpu
def test_user_data_equals_the_host_getter(b200, devshade):
    lib, dev = b200
    host_ud, _ = _host(lib)
    sc, child, keep = _every_kind_with_holes(lib, dev)
    ids = list(range(12)) + [INVALID, 1 << 20]
    t1 = lib.scene_device_traversable(sc)
    lib.check(dev)
    got = _device_user_data(lib, devshade, t1, ids)
    want = []
    for gid in ids:
        w = host_ud(sc, gid)
        lib.rtcGetDeviceError(dev)   # an invalid id records an error on the host
        want.append(w or 0)
    assert got.tolist() == want
    assert want[:8] == [0x1008, 0x2008, 0x3008, 0x4008, 0x5008, 0, 0x7008, 0x8008] and not any(want[8:])
    # a child's data: through the child scene's own traversable
    tc = lib.scene_device_traversable(child)
    assert _device_user_data(lib, devshade, tc, [0]).tolist() == [0x77000]
    # rtcSetGeometryUserData after a getter call: seen by the next traversable without a commit, not by the earlier one
    lib.rtcSetGeometryUserData(lib.rtcGetGeometry(sc, 1), 0xABC0)
    t2 = lib.scene_device_traversable(sc)
    lib.check(dev)
    assert t2.geometries != t1.geometries
    assert _device_user_data(lib, devshade, t2, [1]).tolist() == [0xABC0]
    assert _device_user_data(lib, devshade, t1, [1]).tolist() == [0x2008]
    assert lib.scene_device_traversable(sc).geometries == t2.geometries   # unchanged: the same snapshot
    lib.rtcReleaseScene(sc)
    lib.rtcReleaseScene(child)


@pytest.mark.gpu
def test_user_data_of_a_scene_without_primitives(b200, devshade):
    lib, dev = b200
    v, t = scenes.triangle_sphere(10)
    sc = lib.rtcNewScene(dev)
    keep = lib.add_triangle_mesh(dev, sc, v, t)[1]
    g = lib.rtcGetGeometry(sc, 0)
    lib.rtcSetGeometryUserData(g, 0x5150)
    lib.rtcDisableGeometry(g)
    lib.rtcCommitScene(sc)
    tr = lib.scene_device_traversable(sc)
    lib.check(dev)
    assert tr.root_valid == 0 and tr.geometries
    assert _device_user_data(lib, devshade, tr, [0, 1]).tolist() == [0x5150, 0]
    empty = lib.rtcNewScene(dev)
    lib.rtcCommitScene(empty)
    te = lib.scene_device_traversable(empty)
    lib.check(dev)
    assert not te.geometries and _device_user_data(lib, devshade, te, [0]).tolist() == [0]
    ident = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], np.float32)
    assert (_device_transform(lib, devshade, te, [0], FMT_COL)[0, :12] == ident).all()
    lib.rtcReleaseScene(sc)
    lib.rtcReleaseScene(empty)
    del keep


@pytest.mark.gpu
def test_transforms_equal_the_host_getter(b200, devshade):
    lib, dev = b200
    _, host_xfm = _host(lib)
    rng = np.random.RandomState(15)
    v, t = scenes.triangle_sphere(10)
    child = lib.rtcNewScene(dev)
    keep = [lib.add_triangle_mesh(dev, child, v, t)[1]]
    lib.rtcCommitScene(child)
    sc = lib.rtcNewScene(dev)
    keep.append(lib.add_triangle_mesh(dev, sc, v, t)[1])   # 0: not an instance
    mats = []
    for fmt in (FMT_ROW, FMT_COL, FMT_4X4):                # 1, 2, 3: set through each input format
        m = np.zeros((3, 4), np.float32)
        m[:, :3] = rng.normal(size=(3, 3))
        m[:, 3] = rng.normal(size=3) * 3
        x = {FMT_ROW: m.ravel(), FMT_COL: m.T.ravel(), FMT_4X4: np.concatenate([m, [[0, 0, 0, 1]]]).T.ravel()}[fmt]
        mats.append(m)
        lib.add_instance(dev, sc, child, np.ascontiguousarray(x, np.float32), fmt=fmt)
    lib.rtcCommitScene(sc)
    tr = lib.scene_device_traversable(sc)
    lib.check(dev)
    ids = [0, 1, 2, 3, 4, INVALID]
    for fmt, n in ((FMT_ROW, 12), (FMT_COL, 12), (FMT_4X4, 16)):
        got = _device_transform(lib, devshade, tr, ids, fmt)
        for i, gid in enumerate(ids[:4]):
            w = np.full(16, SENTINEL, np.float32)
            host_xfm(sc, gid, 0.0, fmt, w.ctypes.data)
            lib.check(dev)
            assert got[i].tobytes() == w.tobytes(), (fmt, gid)
        for i in (4, 5):                                   # invalid ids: identity, as geometry 0
            assert got[i].tobytes() == got[0].tobytes(), (fmt, ids[i])
        assert (got[:, n:] == SENTINEL).all()
    assert (_device_transform(lib, devshade, tr, [1, 0], FMT_ROW)[0, :12] == mats[0].ravel()).all()
    assert (_device_transform(lib, devshade, tr, [1, 0, INVALID], RTC_FORMAT_FLOAT) == SENTINEL).all()   # unknown format: untouched
    # a new transform and a re-commit: a new traversable shows it, the old one keeps its snapshot
    m2 = np.array([0, 1, 0, -1, 0, 0, 0, 0, 2, 5, 6, 7], np.float32)
    g = lib.rtcGetGeometry(sc, 2)
    lib.rtcSetGeometryTransform(g, 0, FMT_COL, m2.ctypes.data)
    lib.rtcCommitGeometry(g)
    lib.rtcCommitScene(sc)
    tr2 = lib.scene_device_traversable(sc)
    lib.check(dev)
    assert (_device_transform(lib, devshade, tr2, [2], FMT_COL)[0, :12] == m2).all()
    lib.rtcReleaseScene(sc)
    lib.rtcReleaseScene(child)


# ---- refusals --------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_interpolator_getter_refusals(b200):
    lib, dev = b200
    v, t = scenes.triangle_sphere(10)
    sc = lib.rtcNewScene(dev)
    keep = lib.add_triangle_mesh(dev, sc, v, t)[1]

    def call(bt, slot=0):
        ip = DeviceInterpolator(0x1234, 7, 9)
        n0 = lib.rtcb200GetLaunchCount()
        lib.rtcb200GetSceneDeviceInterpolator(sc, bt, slot, C.byref(ip))
        return lib.rtcGetDeviceError(dev), lib.rtcb200GetLaunchCount() - n0, (ip.table or 0, ip.nentries, ip.reserved)
    assert call(RTC_BUFFER_TYPE_VERTEX) == (3, 0, (0, 0, 0))                 # uncommitted
    lib.rtcCommitScene(sc)
    e, n, (table, nentries, _r) = call(RTC_BUFFER_TYPE_VERTEX)
    assert e == 0 and n == 0 and table and nentries == 1
    assert call(RTC_BUFFER_TYPE_VERTEX)[2][0] == table                         # built once, then shared
    for bt, slot in ((0, 0), (rtc.RTC_BUFFER_TYPE_TANGENT, 0), (RTC_BUFFER_TYPE_VERTEX, 1)):
        assert call(bt, slot) == (3, 0, (0, 0, 0)), (bt, slot)
    assert call(RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 0)[0] == 0                  # a missing slot is a NaN entry, not a refusal
    g = lib.rtcGetGeometry(sc, 0)
    lib.rtcCommitGeometry(g)                                                   # modified: not committed
    assert call(RTC_BUFFER_TYPE_VERTEX) == (3, 0, (0, 0, 0))
    lib.rtcReleaseScene(sc)
    del keep
