"""Seeded rtcInterpolate queries on every curve type, shared by the emulator test (tests/test_interpolate_curves.py), the GPU test
(tests/test_interpolate.py) and the stored reference answers (tests/golden/reference/interpolate_curves.npz).

Each curve type gets one geometry with three buffers -- the FLOAT4 vertex buffer (stride 16), attribute slot 0 (FLOAT4 at a stride of
20 bytes) and attribute slot 1 (FLOAT16 at a stride of 76 bytes, read up to 17 floats) -- and 2002 queries (buffer, valueCount,
primID, u) over the combinations below, u = 0 and u = 1 included."""
import ctypes as C

import numpy as np

from embree_b200.rtc import (InterpolateArguments, RTC_BUFFER_TYPE_INDEX, RTC_BUFFER_TYPE_TANGENT, RTC_BUFFER_TYPE_VERTEX,
                             RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, RTC_FORMAT_FLOAT, RTC_FORMAT_FLOAT4, RTC_FORMAT_UINT, _ptr)

# name -> (RTCGeometryType, rtk::InterpKind for the vertex buffer, for attributes, CurveBasis)
CURVE_TYPES = {
    "round_linear": (16, 3, 3, 0), "flat_linear": (17, 3, 3, 0),
    "round_bezier": (24, 4, 4, 0), "flat_bezier": (25, 4, 4, 0),
    "round_bspline": (32, 4, 4, 1), "flat_bspline": (33, 4, 4, 1),
    "round_hermite": (40, 5, 6, 0), "flat_hermite": (41, 5, 6, 0),
    "round_catmull_rom": (58, 4, 4, 2), "flat_catmull_rom": (59, 4, 4, 2),
}
# buffer -> (bufferType, slot, floats per element as laid out, RTCFormat, valueCounts asked for)
BUFFERS = [(RTC_BUFFER_TYPE_VERTEX, 0, 4, RTC_FORMAT_FLOAT4, (1, 3, 4)),
           (RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 0, 5, RTC_FORMAT_FLOAT4, (1, 3, 4)),
           (RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 1, 19, RTC_FORMAT_FLOAT + 15, (1, 3, 4, 7, 17))]
PER_COMBO = 182   # 11 (buffer, valueCount) combinations per type: 2002 queries
SENTINEL = np.uint32(0x7FC0DEAD).view(np.float32)   # a quiet NaN the reference never computes: marks an output left unwritten


def curve_case(name, seed=0):
    """The geometry and queries of one curve type: dict(verts[n,4], idx, tangents or None, attr0[n,5], attr1[n,19], buf, vc, prim, u)."""
    gtype, _k, _ka, _b = CURVE_TYPES[name]
    rng = np.random.RandomState(1000 + seed + gtype)
    nv = 300
    verts = (rng.normal(size=(nv, 4)) * rng.choice([0.01, 1.0, 50.0], size=(nv, 1))).astype(np.float32)
    verts[:, 3] = np.abs(verts[:, 3]) * 0.1
    span = 1 if "linear" in name or "hermite" in name else 3
    idx = np.sort(rng.choice(nv - span, size=200, replace=False)).astype(np.uint32)
    tangents = (rng.normal(size=(nv, 4)) * 3.0).astype(np.float32) if "hermite" in name else None
    attr0 = rng.normal(size=(nv, 5)).astype(np.float32)
    attr1 = (rng.normal(size=(nv, 19)) * rng.uniform(0.1, 100.0, size=(nv, 1))).astype(np.float32)
    buf, vc = [], []
    for b, (_t, _s, _f, _fmt, counts) in enumerate(BUFFERS):
        for c in counts:
            buf += [b] * PER_COMBO
            vc += [c] * PER_COMBO
    n = len(buf)
    u = rng.uniform(0.0, 1.0, n).astype(np.float32)
    u[0::7] = 0.0
    u[1::7] = 1.0
    u[2::7] = np.float32(1.0) - np.float32(2.0 ** -24) * rng.randint(1, 4, (n + 4) // 7)[: len(u[2::7])]
    return dict(verts=verts, idx=idx, tangents=tangents, attr0=attr0, attr1=attr1, buf=np.array(buf, np.int32), vc=np.array(vc, np.int32),
                prim=rng.randint(0, len(idx), n).astype(np.uint32), u=u)


def make_geometry(L, dev, name, case):
    """The curve geometry of `case` on library L (committed, not attached); returns (geometry, keep-alive list)."""
    gtype = CURVE_TYPES[name][0]
    g = L.rtcNewGeometry(dev, gtype)
    keep = [case["verts"], case["idx"], case["attr0"], case["attr1"]]
    L.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT4, _ptr(case["verts"]), 0, 16, len(case["verts"]))
    L.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT, _ptr(case["idx"]), 0, 4, len(case["idx"]))
    if case["tangents"] is not None:
        L.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_TANGENT, 0, RTC_FORMAT_FLOAT4, _ptr(case["tangents"]), 0, 16, len(case["tangents"]))
        keep.append(case["tangents"])
    L.dll.rtcSetGeometryVertexAttributeCount(C.c_void_p(g), 2)
    for slot, key in ((0, "attr0"), (1, "attr1")):
        _t, _s, floats, fmt, _c = BUFFERS[1 + slot]
        L.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, slot, fmt, _ptr(case[key]), 0, 4 * floats, len(case[key]))
    L.rtcCommitGeometry(g)
    return g, keep


def host_answers(L, g, case, dpdu_only=False):
    """rtcInterpolate of every query of `case` on geometry g: flattened P, dPdu, ddPdudu (value k of query q at offs[q] + k), outputs
    prefilled with SENTINEL.  dpdu_only: one call per query that asks for dPdu alone (P and ddPdudu stay SENTINEL)."""
    offs = np.concatenate([[0], np.cumsum(case["vc"])])
    out = {k: np.full(offs[-1], SENTINEL, np.float32) for k in ("P", "dPdu", "ddPdudu")}
    bufs = [(np.full(17, SENTINEL, np.float32)) for _ in range(3)]
    for q in range(len(case["vc"])):
        t, s, _f, _fmt, _c = BUFFERS[case["buf"][q]]
        vc = int(case["vc"][q])
        for b in bufs:
            b[:] = SENTINEL
        P, du, dd = (_ptr(b) for b in bufs)
        a = InterpolateArguments(g, int(case["prim"][q]), float(case["u"][q]), 0.0, t, s, None if dpdu_only else P, du, None,
                                 None if dpdu_only else dd, None, None, vc)
        L.rtcInterpolate(C.byref(a))
        for k, b in zip(("P", "dPdu", "ddPdudu"), bufs):
            out[k][offs[q]:offs[q + 1]] = b[:vc]
    return out
