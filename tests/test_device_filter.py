"""Argument filters in device-side ray queries: include/embree4_b200_device.cuh with RTCIntersectArguments::filter /
RTCOccludedArguments::filter set to a __device__ function (Embree 4's filter_sycl.h), and the per-geometry snapshot that
rtcb200GetSceneDeviceTraversable uploads for them.

CPU: a user translation unit whose kernel sets args.filter compiles with -I include only and two of them device-link with
-rdc=true; the new feature flags have the reference's values.  GPU (tests/device_filter/devfilter.cu): the reference's golden
answers for argument filters and for the hair tutorial's transparency filter; every byte of every record equal to the
host-pointer path (rtcb200Intersect1M / rtcb200Occluded1M with the same rule as a host C callback) over the scenes of
tests/test_device_traversal.py; what the filter is handed; the feature-mask and per-geometry gating; the snapshot semantics."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from embree_b200 import rtc, scenes
from embree_b200.rtc import RAY_DTYPE, RAYHIT_DTYPE, RayQueryContext, rays_of
from tests import filter_cases as fc
from tests.test_device_traversal import ARCH, INCLUDE, N_RAYS, ROOT, _dev, _nvcc, _quad_instance_scene, _release, query_rays

DEVFILTER = os.path.join(ROOT, "tests", "device_filter", "_build", "libdevfilter.so")
F_NONE, F_ACCEPT, F_RULE, F_EDIT, F_RECORD, F_HAIR, F_HAIR_ID, F_TFAR = range(8)   # devfilter.cu enum Filter
INVOKE = rtc.RTC_RAY_QUERY_FLAG_INVOKE_ARGUMENT_FILTER
ALL = rtc.RTC_FEATURE_FLAG_ALL
INVALID = 0xFFFFFFFF
REC_DTYPE = np.dtype([("ray", "<u4", (12,)), ("hit", "<u4", (9,)), ("ctx_inst", "<u4"), ("ctx_instprim", "<u4"), ("index", "<u4"),
                      ("user", "<u8"), ("accepted", "<u4"), ("pad", "<u4", (5,))])   # devfilter.cu Record (128 bytes)

USER_TU = r"""
#include "embree4_b200.h"
#include "embree4_b200_device.cuh"
__device__ void NAME_cutout(const RTCFilterFunctionNArguments* a) {
  const RTCHit* h = (const RTCHit*)a->hit;
  if (h->primID & 1) a->valid[0] = 0;
}
__global__ void NAME_kernel(RTCB200DeviceTraversable t, RTCRayHit* rh, RTCRay* r, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  RTCIntersectArguments ia; rtcInitIntersectArguments(&ia);
  ia.filter = NAME_cutout;
  rtcb200TraversableIntersect1<RTC_FEATURE_FLAG_FILTER_FUNCTION_IN_ARGUMENTS>(t, rh + i, &ia);
  RTCOccludedArguments oa; rtcInitOccludedArguments(&oa);
  oa.filter = NAME_cutout; oa.flags = RTC_RAY_QUERY_FLAG_INVOKE_ARGUMENT_FILTER;
  rtcb200TraversableOccluded1<RTC_FEATURE_FLAG_ALL>(t, r + i, &oa);
}
void NAME_launch(RTCB200DeviceTraversable t, RTCRayHit* rh, RTCRay* r, int n) { NAME_kernel<<<(n + 127) / 128, 128>>>(t, rh, r, n); }
"""


def _user_tu(d, name):
    path = os.path.join(d, name + ".cu")
    with open(path, "w") as f:
        f.write(USER_TU.replace("NAME", name))
    return path


def test_user_translation_unit_with_a_device_filter_compiles_with_the_public_headers_only():
    with tempfile.TemporaryDirectory() as d:
        _nvcc(["-std=c++17", *ARCH, "-I", INCLUDE, "-c", _user_tu(d, "user"), "-o", "user.o"], d)
        assert os.path.getsize(os.path.join(d, "user.o")) > 0


def test_two_translation_units_with_device_filters_device_link():
    with tempfile.TemporaryDirectory() as d:
        for name in ("a", "b"):
            _nvcc(["-std=c++17", *ARCH, "-rdc=true", "-Xcompiler", "-fPIC", "-I", INCLUDE, "-c", _user_tu(d, name), "-o", name + ".o"], d)
        _nvcc([*ARCH, "-rdc=true", "-shared", "-Xcompiler", "-fPIC", "a.o", "b.o", "-o", "libab.so"], d)
        assert os.path.getsize(os.path.join(d, "libab.so")) > 0


def test_filter_feature_flags_have_the_reference_values():
    src = r"""
#include "embree4_b200.h"
_Static_assert(RTC_FEATURE_FLAG_FILTER_FUNCTION_IN_ARGUMENTS == (1 << 24), "in arguments");
_Static_assert(RTC_FEATURE_FLAG_FILTER_FUNCTION_IN_GEOMETRY == (1 << 25), "in geometry");
_Static_assert(RTC_FEATURE_FLAG_FILTER_FUNCTION == ((1 << 24) | (1 << 25)), "both");
_Static_assert(sizeof(struct RTCB200DeviceGeometry) == 16, "table entry");
_Static_assert(sizeof(struct RTCB200DeviceTraversable) == 48, "traversable");
"""
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "flags.c")
        with open(path, "w") as f:
            f.write(src)
        r = subprocess.run(["cc", "-std=c11", "-fsyntax-only", "-I", INCLUDE, path], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        assert r.returncode == 0, r.stdout
    assert rtc.RTC_FEATURE_FLAG_FILTER_FUNCTION_IN_ARGUMENTS == 1 << 24 and rtc.RTC_FEATURE_FLAG_FILTER_FUNCTION_IN_GEOMETRY == 1 << 25
    assert C.sizeof(rtc.DeviceTraversable) == 48 and rtc.DeviceTraversable.geometries.offset == 40   # passed by value: it did not grow


# ---- GPU -----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def devfilter():
    if not os.path.exists(DEVFILTER):
        subprocess.check_call([os.path.join(ROOT, "tests", "device_filter", "build.sh")])
    L = C.CDLL(DEVFILTER)
    P = C.c_void_p
    L.devfilter_query.argtypes = [P, C.c_int, P, C.c_size_t, C.c_int, C.c_uint, C.c_uint, C.c_int, C.c_uint, C.c_uint, P, P, C.c_uint, P, P, P, P]
    L.devfilter_set_host_T_by_id.argtypes = [P]
    assert L.devfilter_record_words() * 4 == REC_DTYPE.itemsize
    return L


def device_query(lib, dev, L, scene, recs, occluded, which, flags=0, feature_mask=ALL, seed=None, record_cap=0, t=None):
    """One devfilter launch over a copy of `recs`: dict of the records it wrote, the recording filter's calls, the hair
    transparency per ray and the context's ids after the query."""
    import torch
    assert seed is not None or which not in (F_RECORD, F_HAIR, F_HAIR_ID), "these filters read the extended per-thread context"
    if t is None:
        t = lib.scene_device_traversable(scene)
        lib.check(dev)
    n = len(recs)
    d = _dev(recs)
    rec = torch.zeros(max(record_cap, 1) * REC_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
    T = torch.zeros(3 * n, dtype=torch.float32, device="cuda")
    after = torch.zeros(2 * n, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()   # the zero fills above run on the current stream, the query on another one
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        p = lambda x: C.c_void_p(x.data_ptr())   # noqa: E731
        assert L.devfilter_query(C.byref(t), int(occluded), p(d), n, which, flags, feature_mask, 0 if seed is None else 1,
                                 *(seed or (INVALID, INVALID)), p(rec) if record_cap else None, p(cnt), record_cap, p(T), None,
                                 p(after), C.c_void_p(st.cuda_stream)) == 0
    st.synchronize()
    lib.check(dev)
    k = int(cnt.item())
    assert k <= record_cap or not record_cap, "recording buffer too small"
    return {"out": d.cpu().numpy().view(RAY_DTYPE if occluded else RAYHIT_DTYPE), "calls": k,
            "records": rec.cpu().numpy().view(REC_DTYPE)[:k] if record_cap else None,
            "T": T.cpu().numpy().reshape(-1, 3), "after": after.cpu().numpy().view(np.uint32).reshape(-1, 2)}


def host_query(lib, scene, recs, occluded, fn, invoke, seed):
    ctx = RayQueryContext(*seed)
    a = lib.args(filter=fn, invoke_argument_filter=invoke, context=ctx)
    return lib.occluded(scene, recs.copy(), "1M", args=a) if occluded else lib.intersect(scene, recs.copy(), "1M", args=a)


def compare_with_host(lib, dev, L, scene, rh, which, host_fn, invoke=True, seed=(INVALID, INVALID)):
    """Device filter versus the host-pointer path, intersect and occluded: every record byte-identical, except a ray whose
    accepted hit has an accepted twin at bit-equal t (both paths' hits are accepted, same t): those are returned."""
    flags = INVOKE if invoke else 0
    got_i = device_query(lib, dev, L, scene, rh, False, which, flags, seed=seed)["out"]
    want_i = host_query(lib, scene, rh, False, host_fn, invoke, seed)
    lib.check(dev)
    a, b = got_i.view(np.uint8).reshape(-1, 96), want_i.view(np.uint8).reshape(-1, 96)
    bad = np.nonzero((a != b).any(1))[0]
    for i in bad:
        g, w = got_i[i], want_i[i]
        assert g["tfar"].view(np.uint32) == w["tfar"].view(np.uint32), (i, g, w)
        for h in (g, w):
            assert h["geomID"] != INVALID and not fc.rejects(int(h["geomID"]), int(h["primID"]), int(h["instID"])), (i, g, w)
    assert len(bad) <= max(8, len(rh) // 20000), (len(bad), got_i[bad[:4]], want_i[bad[:4]])
    r = rays_of(rh)
    got_o = device_query(lib, dev, L, scene, r, True, which, flags, seed=seed)["out"]
    want_o = host_query(lib, scene, r, True, host_fn, invoke, seed)
    lib.check(dev)
    assert got_o.tobytes() == want_o.tobytes(), np.nonzero((got_o.view(np.uint8).reshape(-1, 48) != want_o.view(np.uint8).reshape(-1, 48)).any(1))[0][:8]
    hits = want_i["geomID"] != INVALID
    assert hits.sum() > len(rh) // 20 and (~hits).sum() > 0
    return got_i, bad


def host_fns(L):
    return {F_RULE: C.cast(L.devfilter_host_rule, C.c_void_p).value, F_EDIT: C.cast(L.devfilter_host_edit, C.c_void_p).value,
            F_TFAR: C.cast(L.devfilter_host_tfar, C.c_void_p).value}


def _host_filter(L, which):
    return rtc.FILTER_FUNCTION(host_fns(L)[which])


# ---- golden answers of the reference ---------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cfg", ["argument_all", "argument_enabled"])
def test_argument_filters_match_the_reference(b200, devfilter, cfg):
    from tests.conftest import load_golden
    from tests.parity import compare_hits
    from tests.test_filter import _golden
    lib, dev = b200
    meshes, rin, _wi, _wo, _b = load_golden("cube_ground")
    want_i, want_o = _golden(cfg)
    last = max(g for (_v, _t, g, _m) in meshes)

    def setup(L, gid, g):
        if cfg == "argument_enabled" and gid == last:
            L.rtcSetGeometryEnableFilterFunctionFromArguments(g, True)
    sc, keep = fc.build(lib, dev, meshes, setup)
    flags = INVOKE if cfg == "argument_all" else 0
    rh = fc.number_rays(rin.copy())
    got_i = device_query(lib, dev, devfilter, sc, rh, False, F_RULE, flags, seed=(INVALID, INVALID))["out"]
    got_o = device_query(lib, dev, devfilter, sc, rays_of(rh), True, F_RULE, flags, seed=(INVALID, INVALID))["out"]
    rep = compare_hits(want_i, got_i, 1e-4, meshes=meshes)
    assert rep["id_mismatch"] == 0 and rep["hit_miss_disagree"] == 0 and rep["tie"] <= 2, (cfg, rep)
    assert rep["max_rel_t"] <= 1e-4 and rep["max_abs_uv"] <= 1e-4 and rep["miss_untouched"], (cfg, rep)
    assert (got_o["tfar"].view(np.uint32) == want_o["tfar"].view(np.uint32)).all(), cfg
    lib.rtcReleaseScene(sc)


@pytest.mark.gpu
def test_hair_shadow_transparency_filter_matches_the_reference(b200, devfilter):
    """hair_geometry_device.cpp:208-262: the occlusion filter multiplies the transparency kept in the caller's extended context
    (one per thread) by the hair's and rejects the hit while more than 2 % is left; only the hair enables the filter."""
    lib, dev = b200
    z = np.load(os.path.join(ROOT, "tests", "golden", "filters.npz"))
    (v, t), (cv, ci), rays = fc.hair_scene()
    sc = lib.rtcNewScene(dev)
    keep = [lib.add_triangle_mesh(dev, sc, v, t, geom_id=0)[1], lib.add_flat_cubic_curves(dev, sc, cv, ci, "bezier", geom_id=1)[1]]
    lib.rtcSetGeometryEnableFilterFunctionFromArguments(lib.rtcGetGeometry(sc, 1), True)
    lib.rtcCommitScene(sc)
    lib.check(dev)
    r = device_query(lib, dev, devfilter, sc, rays, True, F_HAIR, seed=(INVALID, INVALID))
    occ = r["out"]["tfar"] < 0
    T = np.where(occ[:, None], np.float32(0), r["T"])
    assert (occ == z["hair_occluded"]).all()
    assert np.allclose(T, z["hair_T"], rtol=1e-5, atol=1e-7)
    assert 0 < occ.sum() < len(occ) and (T[~occ] < 1).any()
    lib.rtcReleaseScene(sc)
    del keep


# ---- device filter versus the host-pointer path ----------------------------------------------------------------------------
def _sphere_pair(lib, dev, quality, robust):
    sc = lib.rtcNewScene(dev)
    lib.rtcSetSceneFlags(sc, 4 if robust else 0)
    lib.rtcSetSceneBuildQuality(sc, quality)
    v, t = scenes.triangle_sphere(400)
    v2, t2 = scenes.triangle_sphere(60, center=(0.3, 0.2, -0.1), radius=0.4)
    keep = [lib.add_triangle_mesh(dev, sc, v, t, mask=1)[1], lib.add_triangle_mesh(dev, sc, v2, t2, mask=2)[1]]
    lib.rtcCommitScene(sc)
    lib.check(dev)
    return sc, keep


@pytest.mark.gpu
@pytest.mark.parametrize("robust", [False, True])
@pytest.mark.parametrize("quality", [0, 1])
def test_triangle_sphere_pair_matches_the_host_path(b200, devfilter, quality, robust):
    lib, dev = b200
    sc, keep = _sphere_pair(lib, dev, quality, robust)
    rh = query_rays(N_RAYS, (0, 0, 0), 2.0)
    out = {}
    for which in (F_RULE, F_EDIT, F_TFAR):
        out[which], bad = compare_with_host(lib, dev, devfilter, sc, rh, which, _host_filter(devfilter, which))
    # the filter's ray.tfar is what is written: one ulp short of the accepted candidate's t
    hit = (out[F_RULE]["geomID"] != INVALID) & (out[F_RULE]["primID"] == out[F_TFAR]["primID"]) & (out[F_RULE]["geomID"] == out[F_TFAR]["geomID"])
    assert hit.sum() > len(rh) // 20
    assert (out[F_TFAR]["tfar"][hit] == np.nextafter(out[F_RULE]["tfar"][hit], np.float32(0))).all()
    _release(lib, sc)


@pytest.mark.gpu
@pytest.mark.parametrize("robust", [False, True])
def test_quads_under_instances_match_the_host_path(b200, devfilter, robust):
    lib, dev = b200
    top, child, keep = _quad_instance_scene(lib, dev, robust)
    rh = query_rays(N_RAYS, (0, 0, 0), 4.0, seed=3)
    for which in (F_TFAR, F_EDIT, F_RULE):
        out, _ = compare_with_host(lib, dev, devfilter, top, rh, which, _host_filter(devfilter, which), seed=(77, 99))
    hit = out["geomID"] != INVALID
    assert ((out["instID"] == 77) & hit).any() and ((out["instID"] < 7) & hit).any()
    _release(lib, top, child)


@pytest.mark.gpu
def test_scene_of_every_kind_matches_the_host_path(b200, devfilter):
    from tests.test_interpolate import mixed_scene
    lib, dev = b200
    top, child, keep = mixed_scene(lib, dev)
    rh = query_rays(N_RAYS, (0, 0, 0), 8.0, seed=5)
    for which in (F_RULE, F_EDIT):
        compare_with_host(lib, dev, devfilter, top, rh, which, _host_filter(devfilter, which))
    _release(lib, top, child)


@pytest.mark.gpu
def test_points_only_scene_matches_the_host_path(b200, devfilter):
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
    rh = query_rays(N_RAYS, (0, 0, 0), 3.0, seed=7)
    for which in (F_RULE, F_EDIT):
        compare_with_host(lib, dev, devfilter, sc, rh, which, _host_filter(devfilter, which))
    _release(lib, sc)


@pytest.mark.gpu
def test_two_level_and_refitted_dynamic_scenes_match_the_host_path(b200, devfilter):
    from tests.test_gpu_parity import _dynamic_meshes
    lib, dev = b200
    meshes = _dynamic_meshes(24)
    sc = lib.rtcNewScene(dev)
    lib.rtcSetSceneFlags(sc, 1)
    bufs = [lib.add_triangle_mesh(dev, sc, v, t, mask=0xFFFFFFFF) for v, t in meshes]
    lib.rtcCommitScene(sc)
    bufs[2][1][0][:len(meshes[2][0]) * 3] += np.float32(0.35)
    g = lib.rtcGetGeometry(sc, 2)
    lib.rtcUpdateGeometryBuffer(g, rtc.RTC_BUFFER_TYPE_VERTEX, 0)
    lib.rtcCommitGeometry(g)
    lib.rtcCommitScene(sc)
    lib.check(dev)
    assert lib.scene_stats(sc).builder == 3
    rh = query_rays(N_RAYS, (0, 0, 0), 5.0, seed=8)
    for which in (F_RULE, F_EDIT):
        compare_with_host(lib, dev, devfilter, sc, rh, which, _host_filter(devfilter, which))
    _release(lib, sc)

    v, t = scenes.triangle_sphere(200)
    sc = lib.rtcNewScene(dev)
    lib.rtcSetSceneFlags(sc, 1)
    _, (vpad, _i) = lib.add_triangle_mesh(dev, sc, v, t, mask=0xFFFFFFFF, quality=3)
    lib.rtcCommitScene(sc)
    vpad[:v.size] = (v * np.float32([1.3, 1.0, 0.8])).ravel()
    g = lib.rtcGetGeometry(sc, 0)
    lib.rtcUpdateGeometryBuffer(g, rtc.RTC_BUFFER_TYPE_VERTEX, 0)
    lib.rtcCommitGeometry(g)
    lib.rtcCommitScene(sc)
    lib.check(dev)
    assert lib.scene_stats(sc).builder == 2
    rh = query_rays(N_RAYS, (0, 0, 0), 2.5, seed=9)
    for which in (F_RULE, F_EDIT):
        compare_with_host(lib, dev, devfilter, sc, rh, which, _host_filter(devfilter, which))
    _release(lib, sc)


# ---- what the filter is handed -----------------------------------------------------------------------------------------------
def _set_user_data(lib, top, child):
    """Distinct user data on every geometry of `top` and of the `child` it instances: {(scene tag, geomID): value}."""
    a = lib.scene_arrays(top)["descs"]
    ud = {}
    for tag, sc, ids in (("top", top, sorted({int(d["geomID"]) for d in a if d["instID"] == INVALID})),
                         ("child", child, sorted({int(d["geomID"]) for d in a if d["instID"] != INVALID}))):
        for gid in ids:
            ud[(tag, gid)] = 0x10000 * (2 if tag == "child" else 1) + 16 * gid + 8
            lib.rtcSetGeometryUserData(lib.rtcGetGeometry(sc, gid), ud[(tag, gid)])
    return ud


def _check_records(rh, out, r, ud, seed, inst_ids):
    rec = r["records"]
    assert len(rec) > len(rh) // 10
    idx = rec["index"].astype(np.int64)
    ray_in = rh.view(np.uint32).reshape(-1, 24)[idx, :12]
    keep = [0, 1, 2, 3, 4, 5, 6, 7, 9, 10, 11]   # org, tnear, dir, time, mask, id, flags: the caller's ray
    assert (rec["ray"][:, keep] == ray_in[:, keep]).all()
    t = rec["ray"][:, 8].view(np.float32)
    assert (t <= rh["tfar"][idx]).all() and (t >= rh["tnear"][idx]).all()
    geom, inst = rec["hit"][:, 6], rec["hit"][:, 7]
    instanced = np.isin(inst, inst_ids)
    want_user = np.array([ud[("child" if i else "top", int(g))] for g, i in zip(geom, instanced)], np.uint64)
    assert (rec["user"] == want_user).all()
    assert (rec["ctx_inst"] == inst).all() and (rec["ctx_instprim"] == rec["hit"][:, 8]).all()   # instance ids during the call
    assert (rec["hit"][instanced, 8] == 0).all() and (rec["hit"][~instanced, 7] == seed[0]).all()
    assert (r["after"] == np.array(seed, np.uint32)).all()   # and the caller's seed again afterwards
    # the accepted call of every hit ray is the hit written, at the written tfar
    acc = rec[rec["accepted"] == 1]
    seen = {(int(a["index"]), int(a["hit"][5]), int(a["hit"][6]), int(a["hit"][7]), int(a["ray"][8])) for a in acc}
    hit = np.nonzero(out["geomID"] != INVALID)[0]
    assert len(hit) > len(rh) // 20
    for i in hit:
        o = out[i]
        assert (int(i), int(o["primID"]), int(o["geomID"]), int(o["instID"]), int(o["tfar"].view(np.uint32))) in seen, (i, o)


@pytest.mark.gpu
def test_what_the_filter_sees(b200, devfilter):
    from tests.test_interpolate import mixed_scene
    lib, dev = b200
    top, child, keep = mixed_scene(lib, dev)
    ud = _set_user_data(lib, top, child)
    inst_ids = np.array(sorted({int(d["instID"]) for d in lib.scene_arrays(top)["descs"] if d["instID"] != INVALID}), np.uint32)
    assert len(inst_ids) == 6
    rh = query_rays(1 << 18, (0, 0, 0), 8.0, seed=21)
    seed = (5000, 6000)
    r = device_query(lib, dev, devfilter, top, rh, False, F_RECORD, INVOKE, seed=seed, record_cap=8 << 20)
    _check_records(rh, r["out"], r, ud, seed, inst_ids)
    assert len({int(g) for g in r["records"]["hit"][:, 6]}) >= 10
    ro = device_query(lib, dev, devfilter, top, rays_of(rh), True, F_RECORD, INVOKE, seed=seed, record_cap=8 << 20)
    assert ro["calls"] > 0 and (ro["after"] == np.array(seed, np.uint32)).all()
    # an occlusion filter is handed the candidate's hit too: its Ng / ids are those intersect would write for that record
    assert (ro["records"]["hit"][:, 6] != INVALID).all() and (np.abs(ro["records"]["hit"][:, :3].view(np.float32)).sum(1) > 0).any()
    _release(lib, top, child)


@pytest.mark.gpu
def test_triangle_candidates_are_offered_once(b200, devfilter):
    lib, dev = b200
    sc, keep = _sphere_pair(lib, dev, 1, False)
    rh = query_rays(1 << 18, (0, 0, 0), 2.0, seed=22)
    for occluded in (False, True):
        r = device_query(lib, dev, devfilter, sc, rays_of(rh) if occluded else rh, occluded, F_RECORD, INVOKE, seed=(INVALID, INVALID),
                         record_cap=8 << 20)
        rec = r["records"]
        key = rec["index"].astype(np.uint64) << np.uint64(32) | (rec["hit"][:, 6].astype(np.uint64) << np.uint64(24)) | rec["hit"][:, 5]
        assert len(rec) > 1000 and len(np.unique(key)) == len(rec)
    _release(lib, sc)


# ---- gating ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_feature_mask_and_geometry_enable_gate_the_filter(b200, devfilter):
    import torch
    lib, dev = b200
    top, child, keep = _quad_instance_scene(lib, dev, False)
    rh = query_rays(1 << 18, (0, 0, 0), 4.0, seed=23)
    # feature_mask without FILTER_FUNCTION_IN_ARGUMENTS: no call, the unfiltered query's records
    mask = ALL & ~rtc.RTC_FEATURE_FLAG_FILTER_FUNCTION_IN_ARGUMENTS
    for occluded, recs in ((False, rh), (True, rays_of(rh))):
        r = device_query(lib, dev, devfilter, top, recs, occluded, F_RECORD, INVOKE, feature_mask=mask, seed=(INVALID, INVALID), record_cap=1 << 16)
        assert r["calls"] == 0
        want = _dev(recs)
        (lib.rtcb200Occluded1MDevice if occluded else lib.rtcb200Intersect1MDevice)(top, C.c_void_p(want.data_ptr()), len(recs), None, None)
        torch.cuda.synchronize()
        assert r["out"].tobytes() == want.cpu().numpy().tobytes()
    # without INVOKE_ARGUMENT_FILTER: only the geometry that enabled the arguments' filter (the instanced child) is offered
    lib.rtcSetGeometryEnableFilterFunctionFromArguments(lib.rtcGetGeometry(child, 0), True)
    r = device_query(lib, dev, devfilter, top, rh, False, F_RECORD, 0, seed=(INVALID, INVALID), record_cap=8 << 20)
    assert r["calls"] > 1000 and (r["records"]["hit"][:, 7] != INVALID).all()
    both = device_query(lib, dev, devfilter, top, rh, False, F_RECORD, INVOKE, seed=(INVALID, INVALID), record_cap=8 << 20)
    assert (both["records"]["hit"][:, 7] == INVALID).any()
    _release(lib, top, child)


# ---- snapshot semantics ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_traversable_keeps_its_snapshot_of_user_data_and_filter_switch(b200, devfilter):
    lib, dev = b200
    sc, keep = _sphere_pair(lib, dev, 1, False)
    g0, g1 = lib.rtcGetGeometry(sc, 0), lib.rtcGetGeometry(sc, 1)
    lib.rtcSetGeometryUserData(g0, 0x100)
    lib.rtcSetGeometryUserData(g1, 0x200)
    lib.rtcSetGeometryEnableFilterFunctionFromArguments(g1, True)
    t1 = lib.scene_device_traversable(sc)
    assert lib.scene_device_traversable(sc).geometries == t1.geometries   # unchanged: the same snapshot
    lib.rtcSetGeometryUserData(g0, 0x300)
    lib.rtcSetGeometryEnableFilterFunctionFromArguments(g0, True)
    lib.rtcSetGeometryEnableFilterFunctionFromArguments(g1, False)
    t2 = lib.scene_device_traversable(sc)
    lib.check(dev)
    assert t2.geometries != t1.geometries and t2.nodes == t1.nodes
    rh = query_rays(1 << 16, (0, 0, 0), 2.0, seed=24)
    r1 = device_query(lib, dev, devfilter, sc, rh, False, F_RECORD, 0, seed=(INVALID, INVALID), record_cap=1 << 20, t=t1)["records"]
    r2 = device_query(lib, dev, devfilter, sc, rh, False, F_RECORD, 0, seed=(INVALID, INVALID), record_cap=1 << 20, t=t2)["records"]
    assert len(r1) > 100 and (r1["hit"][:, 6] == 1).all() and (r1["user"] == 0x200).all()
    assert len(r2) > 100 and (r2["hit"][:, 6] == 0).all() and (r2["user"] == 0x300).all()
    _release(lib, sc)
