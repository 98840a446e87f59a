"""rtcInterpolate on curves and the batched rtcb200InterpolateHits / rtcb200InterpolateHitsDevice on the GPU.

Host rtcInterpolate on every curve type against the unmodified reference's answers; device interpolation of traced hits against the
host rtcInterpolateN of every hit, bit for bit, in a scene of every supported kind with instances; dynamic and instanced re-commits;
element offsets beyond 2^32; refused arguments; and device memory across repeated commit + interpolate cycles."""
import ctypes as C

import numpy as np
import pytest

from embree_b200 import scenes
from embree_b200.rtc import (INTERP_OUTPUTS, InterpolateHitsArguments, InterpolateNArguments, RAYHIT_DTYPE, RTC_BUFFER_TYPE_INDEX,
                             RTC_BUFFER_TYPE_TANGENT, RTC_BUFFER_TYPE_VERTEX, RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, RTC_FORMAT_FLOAT,
                             RTC_FORMAT_FLOAT3, RTC_FORMAT_FLOAT4, RTC_FORMAT_UINT, RTC_FORMAT_UINT3, RTC_FORMAT_UINT4, _ptr, make_rayhits)
from tests.interp_cases import BUFFERS, CURVE_TYPES, SENTINEL, curve_case, host_answers, make_geometry
from tests.test_interpolate_curves import LINEAR, reference_curve_answers

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


def test_host_curve_interpolation_matches_the_reference(b200):
    """rtcInterpolate on every curve type gives the reference's bits (linear curves: the documented ddPdudu difference); rtcInterpolateN
    gives the same values and 0 in the v-derivatives."""
    lib, dev = b200
    ref = reference_curve_answers()
    for name in CURVE_TYPES:
        case = curve_case(name)
        g, keep = make_geometry(lib, dev, name, case)
        mine = host_answers(lib, g, case)
        lib.check(dev)
        assert (mine["P"].view(np.uint32) == ref[name]["P"].view(np.uint32)).all(), name
        if name in LINEAR:
            assert (mine["dPdu"].view(np.uint32) == ref[name]["dPdu_alone"].view(np.uint32)).all() and (mine["ddPdudu"] == 0).all()
        else:
            for k in ("dPdu", "ddPdudu"):
                assert (mine[k].view(np.uint32) == ref[name][k].view(np.uint32)).all(), (name, k)
        # rtcInterpolateN over the queries of attribute slot 1 with valueCount 7
        q = np.nonzero((case["buf"] == 2) & (case["vc"] == 7))[0]
        out = {k: np.full((7, len(q)), SENTINEL, np.float32) for k in INTERP_OUTPUTS}
        prim, u, v = np.ascontiguousarray(case["prim"][q]), np.ascontiguousarray(case["u"][q]), np.zeros(len(q), np.float32)
        a = InterpolateNArguments(g, None, prim.ctypes.data, u.ctypes.data, v.ctypes.data, len(q), RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 1,
                                  *[out[k].ctypes.data for k in INTERP_OUTPUTS], 7)
        lib.rtcInterpolateN(C.byref(a))
        lib.check(dev)
        offs = np.concatenate([[0], np.cumsum(case["vc"])])
        for j, qi in enumerate(q):
            assert (out["P"][:, j].view(np.uint32) == mine["P"][offs[qi]:offs[qi + 1]].view(np.uint32)).all()
        assert not out["dPdv"].any() and not out["ddPdvdv"].any() and not out["ddPdudv"].any()
        lib.rtcReleaseGeometry(g)


# ---- scenes ------------------------------------------------------------------------------------------------------------
def add_geometry(L, dev, scene, gtype, verts, idx, tangents=None, attrs=(), keep=None, tstride=16):
    """A geometry of any supported kind with shared buffers: `attrs` = [(array[n, floats], RTCFormat, byte stride)] attribute slots."""
    g = L.rtcNewGeometry(dev, gtype)
    keep.append([verts, idx, tangents] + [a for a, _f, _s in attrs])
    v4 = verts.shape[1] == 4
    L.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT4 if v4 else RTC_FORMAT_FLOAT3, _ptr(verts), 0, 4 * verts.shape[1] if v4 else 12,
                                 len(verts) if v4 else len(verts) - 1)
    if idx is not None:
        fmt = {1: RTC_FORMAT_UINT, 3: RTC_FORMAT_UINT3, 4: RTC_FORMAT_UINT4}[1 if idx.ndim == 1 else idx.shape[1]]
        L.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_INDEX, 0, fmt, _ptr(idx), 0, idx.itemsize * (1 if idx.ndim == 1 else idx.shape[1]), len(idx))
    if tangents is not None:
        L.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_TANGENT, 0, RTC_FORMAT_FLOAT4, _ptr(tangents), 0, tstride, len(verts))
    if attrs:
        L.dll.rtcSetGeometryVertexAttributeCount(C.c_void_p(g), len(attrs))
        for slot, (a, fmt, stride) in enumerate(attrs):
            L.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, slot, fmt, _ptr(a), 0, stride, len(verts) - (0 if v4 else 1))
    L.rtcCommitGeometry(g)
    gid = L.rtcAttachGeometry(scene, g)
    L.rtcReleaseGeometry(g)
    return gid


def attrs_for(rng, n):
    """slot 0: FLOAT3 at a 20-byte stride (scalar loads); slot 1: FLOAT4 at 16 bytes (16-byte loads)"""
    return [(rng.normal(size=(n, 5)).astype(np.float32), RTC_FORMAT_FLOAT3, 20), (rng.normal(size=(n, 4)).astype(np.float32), RTC_FORMAT_FLOAT4, 16)]


def fill_kinds(L, dev, scene, rng, keep, scale=1.0):
    """A triangle sphere, a quad grid, all ten curve types, sphere points and a triangle mesh without attributes."""
    v, t = scenes.triangle_sphere(40)
    v = np.concatenate([v * np.float32(0.8 * scale), np.zeros((1, 3), np.float32)]).astype(np.float32)   # one float of padding
    add_geometry(L, dev, scene, 0, v, t, attrs=attrs_for(rng, len(v)), keep=keep)
    n = 12
    gx, gy = np.meshgrid(np.linspace(-2, 2, n + 1), np.linspace(-2, 2, n + 1))
    qv = np.concatenate([np.stack([gx.ravel(), gy.ravel(), np.full(gx.size, -1.2)], 1) * scale, np.zeros((1, 3))]).astype(np.float32)
    a = np.arange(n * (n + 1)).reshape(n, n + 1)[:, :n].ravel()
    qi = np.stack([a, a + 1, a + n + 2, a + n + 1], 1).astype(np.uint32)
    add_geometry(L, dev, scene, 1, qv, qi, attrs=attrs_for(rng, len(qv)), keep=keep)
    for name, (gtype, _kv, _ka, _b) in CURVE_TYPES.items():
        if "linear" in name:
            cv, ci, _ = scenes.hair_ball(300, 4, seed=gtype, radius=0.8 * scale, length=0.6 * scale, width=0.04 * scale)
            tg = None
        else:
            basis = name.split("_", 1)[1]
            cv, ci, tg = scenes.cubic_hair(150, basis, knots=7, seed=gtype, radius=0.8 * scale, step=0.12 * scale, width=0.03 * scale)
        cv = np.ascontiguousarray(cv, np.float32)
        ts = 32
        if tg is not None:   # tangents at their own stride, which differs from the vertex buffer's
            tgw = np.zeros((len(tg), 8), np.float32)
            tgw[:, :4] = tg
            tg = tgw
        add_geometry(L, dev, scene, gtype, cv, np.ascontiguousarray(ci, np.uint32), tangents=tg, attrs=attrs_for(rng, len(cv)), keep=keep,
                     tstride=ts)
    pv = np.concatenate([rng.normal(size=(200, 3)) * 0.9 * scale, rng.uniform(0.03, 0.08, (200, 1)) * scale], 1).astype(np.float32)
    add_geometry(L, dev, scene, 50, pv, None, attrs=attrs_for(rng, len(pv)), keep=keep)
    v2, t2 = scenes.triangle_sphere(20)
    v2 = np.concatenate([v2 * np.float32(0.3 * scale) + np.float32(0.9 * scale), np.zeros((1, 3), np.float32)]).astype(np.float32)
    add_geometry(L, dev, scene, 0, v2, t2, keep=keep)      # no attribute slots


def mixed_scene(L, dev, seed=5):
    rng = np.random.RandomState(seed)
    keep = []
    child = L.rtcNewScene(dev)
    fill_kinds(L, dev, child, rng, keep, scale=0.5)
    L.rtcCommitScene(child)
    top = L.rtcNewScene(dev)
    fill_kinds(L, dev, top, rng, keep)
    for i in range(6):
        q, _r = np.linalg.qr(rng.normal(size=(3, 3)))
        m = (q * rng.uniform(0.6, 1.4, 3)[None, :]).astype(np.float32)
        p = (rng.normal(size=3) * 3.0).astype(np.float32)
        L.add_instance(dev, top, child, np.concatenate([m[:, 0], m[:, 1], m[:, 2], p]).astype(np.float32))
    L.rtcCommitScene(top)
    L.check(dev)
    return top, child, keep


def rays(n, seed=9, spread=4.0):
    rng = np.random.RandomState(seed)
    o = rng.normal(size=(n, 3))
    o = (o / np.linalg.norm(o, axis=1, keepdims=True) * 8.0).astype(np.float32)
    tgt = rng.uniform(-spread, spread, (n, 3)).astype(np.float32)
    return make_rayhits(o, tgt - o)


def host_interpolate(L, dev, scene, child, hits, bt, slot, vc):
    """The host rtcInterpolateN of every hit, grouped by geometry (`child`: the scene the instances instantiate): {name: [vc, M]}
    (misses and geometries it refuses stay NaN) and the mask of the hits whose geometry it refused."""
    M = len(hits)
    out = {k: np.full((vc, M), np.nan, np.float32) for k in INTERP_OUTPUTS}
    refused = np.zeros(M, bool)
    hit = hits["geomID"] != 0xFFFFFFFF
    keys = np.stack([hits["instID"], hits["geomID"]], 1)
    for inst, gid in np.unique(keys[hit], axis=0):
        sel = np.nonzero(hit & (hits["instID"] == inst) & (hits["geomID"] == gid))[0]
        sc = scene if inst == 0xFFFFFFFF else child
        g = L.rtcGetGeometry(sc, int(gid))
        prim, u, v = (np.ascontiguousarray(hits[f][sel]) for f in ("primID", "u", "v"))
        o = {k: np.full((vc, len(sel)), np.nan, np.float32) for k in INTERP_OUTPUTS}
        a = InterpolateNArguments(g, None, prim.ctypes.data, u.ctypes.data, v.ctypes.data, len(sel), bt, slot,
                                  *[o[k].ctypes.data for k in INTERP_OUTPUTS], vc)
        L.rtcInterpolateN(C.byref(a))
        if L.rtcGetDeviceError(dev) != 0:
            refused[sel] = True
            continue
        for k in INTERP_OUTPUTS:
            out[k][:, sel] = o[k]
    return out, refused


def device_hits(lib, scene, r, stream):
    d = torch.from_numpy(r.view(np.uint8).copy()).cuda()
    with torch.cuda.stream(stream):
        lib.rtcb200Intersect1MDevice(scene, C.c_void_p(d.data_ptr()), len(r), C.byref(lib.args()), C.c_void_p(stream.cuda_stream))
    return d


def test_mixed_scene_device_interpolation_matches_host(b200):
    lib, dev = b200
    top, child, keep = mixed_scene(lib, dev)
    r = rays(1 << 20)
    st = torch.cuda.Stream()
    d = device_hits(lib, top, r, st)
    for bt, slot, vc in ((RTC_BUFFER_TYPE_VERTEX, 0, 3), (RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 0, 3), (RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 1, 4)):
        sentinel = {k: torch.full((vc, len(r)), -7.5, dtype=torch.float32, device="cuda") for k in INTERP_OUTPUTS}
        got = lib.interpolate_hits(top, d, bt, slot, vc, want=INTERP_OUTPUTS, stream=st, out=sentinel)   # same stream, no sync between
        lib.check(dev)
        hits = d.cpu().numpy().view(RAYHIT_DTYPE).reshape(-1)
        want, refused = host_interpolate(lib, dev, top, child, hits, bt, slot, vc)
        hit = hits["geomID"] != 0xFFFFFFFF
        kinds = set(zip(hits["instID"][hit].tolist(), hits["geomID"][hit].tolist()))
        assert len(kinds) >= 20 and refused.any() and (hits["instID"] != 0xFFFFFFFF).any(), len(kinds)
        for k in INTERP_OUTPUTS:
            g = got[k].cpu().numpy()
            assert (g[:, ~hit] == -7.5).all(), k                                          # misses untouched
            assert np.isnan(g[:, refused]).all(), k                                       # points and the missing slot: NaN
            ok = hit & ~refused
            assert (g[:, ok].view(np.uint32) == want[k][:, ok].view(np.uint32)).all(), k
        # curves: zero v-derivatives
        curve = ok & np.isin(hits["geomID"], np.arange(2, 12))
        assert curve.sum() > 1000 and not got["dPdv"].cpu().numpy()[:, curve].any()
        # the host-pointer variant gives the same bits
        hv = lib.interpolate_hits(top, hits.copy(), bt, slot, vc, want=INTERP_OUTPUTS)
        for k in INTERP_OUTPUTS:
            g = got[k].cpu().numpy()
            assert (np.where(hit, hv[k], -7.5).view(np.uint32) == g.view(np.uint32)).all(), k
    lib.rtcReleaseScene(top)
    lib.rtcReleaseScene(child)


def test_dynamic_and_instanced_recommit(b200):
    """A two-level dynamic scene sees moved vertices after the re-commit; an attribute edit is seen after rtcUpdateGeometryBuffer and the
    commits, through a re-committed instanced scene too."""
    lib, dev = b200
    rng = np.random.RandomState(2)
    keep = []
    sc = lib.rtcNewScene(dev)
    lib.rtcSetSceneFlags(sc, 1)
    meshes = []
    for i in range(3):
        v, t = scenes.triangle_sphere(30, center=(3.0 * i - 3.0, 0.0, 0.0))
        v = np.concatenate([v, np.zeros((1, 3), np.float32)]).astype(np.float32)
        meshes.append(v)
        add_geometry(lib, dev, sc, 0, v, t, attrs=[(rng.normal(size=(len(v), 4)).astype(np.float32), RTC_FORMAT_FLOAT4, 16)], keep=keep)
    lib.rtcCommitScene(sc)
    r = make_rayhits(np.stack([rng.uniform(-5, 5, 20000), rng.uniform(-1, 1, 20000), np.full(20000, -5.0)], 1), np.tile([[0, 0, 1]], (20000, 1)))
    hits = lib.intersect(sc, r.copy(), "1M")
    d = torch.from_numpy(hits.view(np.uint8).copy()).cuda()

    def check(scene, bt, slot, vc):
        got = lib.interpolate_hits(scene, d, bt, slot, vc, want=("P",))["P"].cpu().numpy()
        want, refused = host_interpolate(lib, dev, scene, None, hits, bt, slot, vc)
        ok = hits["geomID"] != 0xFFFFFFFF
        assert ok.sum() > 5000 and not refused.any()
        assert (got[:, ok].view(np.uint32) == want["P"][:, ok].view(np.uint32)).all()
        return got
    before = check(sc, RTC_BUFFER_TYPE_VERTEX, 0, 3)
    meshes[1][:-1] += np.float32(0.25)
    g1 = lib.rtcGetGeometry(sc, 1)
    lib.rtcUpdateGeometryBuffer(g1, RTC_BUFFER_TYPE_VERTEX, 0)
    lib.rtcCommitGeometry(g1)
    lib.rtcCommitScene(sc)
    after = check(sc, RTC_BUFFER_TYPE_VERTEX, 0, 3)
    on1 = hits["geomID"] == 1
    assert (after[:, on1] != before[:, on1]).all() and (after[:, ~on1 & (hits["geomID"] != 0xFFFFFFFF)] == before[:, ~on1 & (hits["geomID"] != 0xFFFFFFFF)]).all()
    # attribute edit, direct
    check(sc, RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 0, 4)
    keep[0][3][:] *= np.float32(2.0)
    g0 = lib.rtcGetGeometry(sc, 0)
    lib.rtcUpdateGeometryBuffer(g0, RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 0)
    lib.rtcCommitGeometry(g0)
    lib.rtcCommitScene(sc)
    check(sc, RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 0, 4)
    # through an instance: the child is re-committed, then the scene that instances it
    top = lib.rtcNewScene(dev)
    lib.add_instance(dev, top, sc, np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], np.float32))
    lib.rtcCommitScene(top)
    ihits = lib.intersect(top, r.copy(), "1M")
    assert (ihits["instID"][ihits["geomID"] != 0xFFFFFFFF] == 0).all()
    di = torch.from_numpy(ihits.view(np.uint8).copy()).cuda()
    first = lib.interpolate_hits(top, di, RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 0, 4, want=("P",))["P"].cpu().numpy()
    keep[1][3][:] += np.float32(1.0)
    lib.rtcUpdateGeometryBuffer(g1, RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 0)
    lib.rtcCommitGeometry(g1)
    lib.rtcCommitScene(sc)
    a = InterpolateHitsArguments()
    a.hits, a.M, a.bufferType, a.valueCount, a.P = di.data_ptr(), len(ihits), RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 4, first.ctypes.data
    lib.rtcb200InterpolateHits(top, C.byref(a))                 # the instancing scene is modified until it is committed again
    assert lib.rtcGetDeviceError(dev) == 3
    lib.rtcCommitScene(top)
    second = lib.interpolate_hits(top, di, RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 0, 4, want=("P",))["P"].cpu().numpy()
    want, _ = host_interpolate(lib, dev, top, sc, ihits, RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 0, 4)
    ok = ihits["geomID"] != 0xFFFFFFFF
    assert (second[:, ok].view(np.uint32) == want["P"][:, ok].view(np.uint32)).all()
    on1 = ihits["geomID"] == 1
    assert on1.sum() > 1000 and (second[:, on1] != first[:, on1]).all()
    lib.check(dev)
    lib.rtcReleaseScene(top)
    lib.rtcReleaseScene(sc)


def test_large_batches_cross_32_bit_offsets(b200):
    """272 Mi hits x 16 values: value j of hit i at j * M + i passes 2^31 and 2^32.  A strided sample is checked against the host."""
    lib, dev = b200
    keep = []
    sc = lib.rtcNewScene(dev)
    rng = np.random.RandomState(4)
    v, t = scenes.triangle_sphere(60)
    v = np.concatenate([v, np.zeros((1, 3), np.float32)]).astype(np.float32)
    add_geometry(lib, dev, sc, 0, v, t, attrs=[(rng.normal(size=(len(v), 16)).astype(np.float32), RTC_FORMAT_FLOAT + 15, 64)], keep=keep)
    lib.rtcCommitScene(sc)
    M, vc = 272 << 20, 16
    assert M * vc > 2 ** 32
    hits = torch.zeros((M, 24), dtype=torch.int32, device="cuda")
    i = torch.arange(M, device="cuda", dtype=torch.int64)
    hits[:, 15] = (torch.rand(M, device="cuda") * 0.5).view(torch.int32)
    hits[:, 16] = (torch.rand(M, device="cuda") * 0.5).view(torch.int32)
    hits[:, 17] = (i * 2654435761 % len(t)).to(torch.int32)
    hits[:, 18] = 0
    hits[:, 19] = -1
    hits[i % 1009 == 5, 18] = -1                      # some misses
    P = lib.interpolate_hits(sc, hits, RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 0, vc, want=("P",))["P"]
    torch.cuda.synchronize()
    lib.check(dev)
    sample = torch.cat([torch.arange(0, M, 99991, device="cuda"), torch.arange(M - 300, M, device="cuda")])
    h = hits[sample].cpu().numpy().view(RAYHIT_DTYPE).reshape(-1)
    got = P[:, sample].cpu().numpy()
    del P, hits
    want, refused = host_interpolate(lib, dev, sc, None, h, RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 0, vc)
    miss = h["geomID"] == 0xFFFFFFFF
    assert miss.any() and (~miss).sum() > 2000 and not refused.any()
    assert np.isnan(got[:, miss]).all()
    assert (got[:, ~miss].view(np.uint32) == want["P"][:, ~miss].view(np.uint32)).all()
    lib.rtcReleaseScene(sc)
    torch.cuda.empty_cache()


def test_refused_arguments_launch_nothing(b200):
    lib, dev = b200
    keep = []
    sc = lib.rtcNewScene(dev)
    v, t = scenes.triangle_sphere(10)
    v = np.concatenate([v, np.zeros((1, 3), np.float32)]).astype(np.float32)
    add_geometry(lib, dev, sc, 0, v, t, attrs=[(np.ones((len(v), 4), np.float32), RTC_FORMAT_FLOAT3, 16)], keep=keep)
    hits = make_rayhits(np.zeros((4, 3)), np.tile([[0, 0, 1]], (4, 1)))
    hits["geomID"], hits["primID"] = 0, 1
    out = np.zeros(300 * 4, np.float32)

    def call(bt=RTC_BUFFER_TYPE_VERTEX, slot=0, vc=3, dpdu=False, dpdv=False):
        a = InterpolateHitsArguments()
        a.hits, a.M, a.bufferType, a.bufferSlot, a.valueCount, a.P = hits.ctypes.data, 4, bt, slot, vc, out.ctypes.data
        a.dPdu = out.ctypes.data if dpdu else None
        a.dPdv = out.ctypes.data if dpdv else None
        n0 = lib.rtcb200GetLaunchCount()
        lib.rtcb200InterpolateHits(sc, C.byref(a))
        return lib.rtcGetDeviceError(dev), lib.rtcb200GetLaunchCount() - n0
    assert call() == (3, 0)                                          # uncommitted scene
    lib.rtcCommitScene(sc)
    assert call() == (0, 1)
    assert call(vc=257) == (3, 0)
    assert call(dpdu=True) == (2, 0) and call(dpdv=True) == (2, 0)
    assert call(bt=RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, vc=4) == (2, 0)  # FLOAT3 attribute, 4 values
    assert call(bt=RTC_BUFFER_TYPE_VERTEX, slot=1) == (2, 0)
    assert call(bt=RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, vc=3) == (0, 1)
    g = lib.rtcGetGeometry(sc, 0)
    lib.rtcCommitGeometry(g)                                          # modified: not committed
    assert call() == (3, 0)
    lib.rtcReleaseScene(sc)


def test_repeated_commit_and_interpolate_keep_device_memory_flat(b200):
    lib, dev = b200
    keep = []
    sc = lib.rtcNewScene(dev)
    rng = np.random.RandomState(3)
    v, t = scenes.triangle_sphere(200)
    v = np.concatenate([v, np.zeros((1, 3), np.float32)]).astype(np.float32)
    add_geometry(lib, dev, sc, 0, v, t, attrs=attrs_for(rng, len(v)), keep=keep)
    cv, ci, tg = scenes.cubic_hair(2000, "hermite", knots=7, seed=1)
    add_geometry(lib, dev, sc, 40, np.ascontiguousarray(cv, np.float32), np.ascontiguousarray(ci, np.uint32), tangents=np.ascontiguousarray(tg, np.float32),
                 attrs=attrs_for(rng, len(cv)), keep=keep)
    r = rays(1 << 18, spread=1.0)
    d = torch.from_numpy(r.view(np.uint8).copy()).cuda()

    def cycle():
        g = lib.rtcGetGeometry(sc, 0)
        lib.rtcUpdateGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0)
        lib.rtcCommitGeometry(g)
        lib.rtcCommitScene(sc)
        st = torch.cuda.current_stream()
        lib.rtcb200Intersect1MDevice(sc, C.c_void_p(d.data_ptr()), len(r), C.byref(lib.args()), C.c_void_p(st.cuda_stream))
        for bt, slot, vc in ((RTC_BUFFER_TYPE_VERTEX, 0, 3), (RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 0, 3), (RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 1, 4)):
            lib.interpolate_hits(sc, d, bt, slot, vc, want=("P", "dPdu", "dPdv"))
        torch.cuda.synchronize()
        lib.check(dev)
    cycle()
    torch.cuda.empty_cache()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(20):
        cycle()
    torch.cuda.empty_cache()
    free1 = torch.cuda.mem_get_info()[0]
    assert free0 - free1 < 32 << 20, (free0, free1)
    lib.rtcReleaseScene(sc)
