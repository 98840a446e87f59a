"""ctypes mirror of the rtc* C-ABI declared in include/embree4_b200.h.

The same binding class drives ANY library that exports the Embree 4 C API, so the parity tests
read like the reference's own tests (tutorials/verify/rtcore_helpers.h:701-787 `IntersectWithMode`):
the product library (embree_b200/csrc/libembree4_b200.so) and -- in tests/bench only -- the
unmodified reference (oracle/_ref/libembree4.so.4) are loaded through `RTCLib(path)`.

Layouts follow include/embree4/rtcore_ray.h:11-184 (sizeof(RTCRayHit) == 96).
"""
import ctypes as C
import os

import numpy as np

RTC_INVALID_GEOMETRY_ID = 0xFFFFFFFF
RTC_FORMAT_UINT3 = 0x5003
RTC_FORMAT_UINT4 = 0x5004
RTC_FORMAT_FLOAT3 = 0x9003
RTC_BUFFER_TYPE_INDEX = 0
RTC_BUFFER_TYPE_VERTEX = 1
RTC_GEOMETRY_TYPE_TRIANGLE = 0
RTC_GEOMETRY_TYPE_QUAD = 1
RTC_GEOMETRY_TYPE_ROUND_LINEAR_CURVE = 16
RTC_GEOMETRY_TYPE_FLAT_LINEAR_CURVE = 17
RTC_GEOMETRY_TYPE_INSTANCE = 121
RTC_GEOMETRY_TYPE_FLAT_BEZIER_CURVE, RTC_GEOMETRY_TYPE_FLAT_BSPLINE_CURVE = 25, 33
RTC_GEOMETRY_TYPE_FLAT_HERMITE_CURVE, RTC_GEOMETRY_TYPE_FLAT_CATMULL_ROM_CURVE = 41, 59
FLAT_CUBIC_TYPES = {"bezier": 25, "bspline": 33, "hermite": 41, "catmull_rom": 59}
ROUND_CUBIC_TYPES = {"bezier": 24, "bspline": 32, "hermite": 40, "catmull_rom": 58}
RTC_BUFFER_TYPE_TANGENT = 4
RTC_BUFFER_TYPE_NORMAL = 3
POINT_TYPES = {"sphere": 50, "disc": 51, "oriented_disc": 52}   # RTC_GEOMETRY_TYPE_SPHERE_POINT / _DISC_POINT / _ORIENTED_DISC_POINT
RTC_FORMAT_UCHAR = 0x1001
RTC_FORMAT_UINT = 0x5001
RTC_FORMAT_FLOAT4 = 0x9004
RTC_BUFFER_TYPE_FLAGS = 32
RTC_FORMAT_FLOAT3X4_ROW_MAJOR = 0x9134
RTC_FORMAT_FLOAT3X4_COLUMN_MAJOR = 0x9234
RTC_FORMAT_FLOAT4X4_COLUMN_MAJOR = 0x9244
RTC_BUILD_QUALITY_LOW, RTC_BUILD_QUALITY_MEDIUM, RTC_BUILD_QUALITY_HIGH, RTC_BUILD_QUALITY_REFIT = 0, 1, 2, 3
RTC_SCENE_FLAG_NONE, RTC_SCENE_FLAG_DYNAMIC, RTC_SCENE_FLAG_COMPACT, RTC_SCENE_FLAG_ROBUST = 0, 1, 2, 4
RTC_RAY_QUERY_FLAG_INCOHERENT = 0
RTC_RAY_QUERY_FLAG_COHERENT = 1 << 16
RTC_FEATURE_FLAG_ALL = 0xFFFFFFFF
RTC_ERROR_NONE, RTC_ERROR_UNKNOWN, RTC_ERROR_INVALID_ARGUMENT, RTC_ERROR_INVALID_OPERATION = 0, 1, 2, 3

# numpy views of the I/O records ---------------------------------------------------------------
RAYHIT_DTYPE = np.dtype([
    ("org_x", "<f4"), ("org_y", "<f4"), ("org_z", "<f4"), ("tnear", "<f4"),
    ("dir_x", "<f4"), ("dir_y", "<f4"), ("dir_z", "<f4"), ("time", "<f4"),
    ("tfar", "<f4"), ("mask", "<u4"), ("id", "<u4"), ("flags", "<u4"),
    ("Ng_x", "<f4"), ("Ng_y", "<f4"), ("Ng_z", "<f4"), ("u", "<f4"), ("v", "<f4"),
    ("primID", "<u4"), ("geomID", "<u4"), ("instID", "<u4"), ("instPrimID", "<u4"),
    ("pad0", "<u4"), ("pad1", "<u4"), ("pad2", "<u4"),
])
RAY_DTYPE = np.dtype(RAYHIT_DTYPE.descr[:12])
assert RAYHIT_DTYPE.itemsize == 96 and RAY_DTYPE.itemsize == 48

_RAY_FIELDS = ["org_x", "org_y", "org_z", "tnear", "dir_x", "dir_y", "dir_z", "time", "tfar", "mask", "id", "flags"]
_HIT_FIELDS = ["Ng_x", "Ng_y", "Ng_z", "u", "v", "primID", "geomID", "instID", "instPrimID"]


def packet_dtype(K, hit=True):
    """RTCRayHit{K} / RTCRay{K} as a numpy structured dtype (SoA inside one packet)."""
    f = [(n, "<u4" if n in ("mask", "id", "flags") else "<f4", (K,)) for n in _RAY_FIELDS]
    if hit:
        f += [(n, "<f4" if n in ("Ng_x", "Ng_y", "Ng_z", "u", "v") else "<u4", (K,)) for n in _HIT_FIELDS]
    d = np.dtype(f)
    assert d.itemsize == (21 if hit else 12) * 4 * K
    return d


def aligned_empty(n, dtype, align=64):
    """n records of `dtype`, base address aligned (packets need 16/32/64 B: rtcore.cpp:607,679,806,867)."""
    dtype = np.dtype(dtype)
    raw = np.empty(n * dtype.itemsize + align, dtype=np.uint8)
    off = (-raw.ctypes.data) % align
    return raw[off:off + n * dtype.itemsize].view(dtype)


def make_rayhits(org, dir, tnear=0.0, tfar=np.inf, mask=0xFFFFFFFF):
    """Fresh RTCRayHit[] with hit.geomID preset to INVALID as the API contract requires
    (doc/src/api/rtcIntersect1.md:26-44)."""
    org = np.asarray(org, np.float32).reshape(-1, 3)
    dir = np.asarray(dir, np.float32).reshape(-1, 3)
    n = org.shape[0]
    r = aligned_empty(n, RAYHIT_DTYPE)
    r.view(np.uint8)[:] = 0
    r["org_x"], r["org_y"], r["org_z"] = org[:, 0], org[:, 1], org[:, 2]
    r["dir_x"], r["dir_y"], r["dir_z"] = dir[:, 0], dir[:, 1], dir[:, 2]
    r["tnear"] = tnear
    r["tfar"] = tfar
    r["mask"] = mask
    r["id"] = np.arange(n, dtype=np.uint32)
    r["geomID"] = RTC_INVALID_GEOMETRY_ID
    r["primID"] = RTC_INVALID_GEOMETRY_ID
    r["instID"] = RTC_INVALID_GEOMETRY_ID
    r["instPrimID"] = RTC_INVALID_GEOMETRY_ID
    return r


def rays_of(rayhits):
    """Copy the RTCRay halves of RTCRayHit[] into a contiguous RTCRay[] (for rtcOccluded*)."""
    out = aligned_empty(len(rayhits), RAY_DTYPE)
    for f in _RAY_FIELDS:
        out[f] = rayhits[f]
    return out


def to_packets(rayhits, K, hit=True):
    """AoS RTCRayHit[] -> RTCRayHit{K}[] (+ valid mask, -1 active / 0 padding)."""
    n = len(rayhits)
    m = (n + K - 1) // K
    p = aligned_empty(m, packet_dtype(K, hit))
    p.view(np.uint8)[:] = 0
    valid = aligned_empty(m * K, np.int32)
    valid[:] = 0
    valid[:n] = -1
    for f in _RAY_FIELDS + (_HIT_FIELDS if hit else []):
        flat = np.zeros(m * K, dtype=rayhits.dtype[f] if f in rayhits.dtype.names else np.uint32)
        flat[:n] = rayhits[f]
        p[f] = flat.reshape(m, K)
    return p, valid


def from_packets(p, n, hit=True):
    K = p.dtype["org_x"].shape[0]
    out = aligned_empty(n, RAYHIT_DTYPE if hit else RAY_DTYPE)
    out.view(np.uint8)[:] = 0
    for f in _RAY_FIELDS + (_HIT_FIELDS if hit else []):
        out[f] = p[f].reshape(-1)[:n]
    return out


class _IntersectArguments(C.Structure):
    _fields_ = [("flags", C.c_uint), ("feature_mask", C.c_uint), ("context", C.c_void_p),
                ("filter", C.c_void_p), ("intersect", C.c_void_p)]


class RayQueryContext(C.Structure):
    _fields_ = [("instID", C.c_uint), ("instPrimID", C.c_uint)]


class FilterFunctionNArguments(C.Structure):
    """RTCFilterFunctionNArguments (rtcore_common.h:311-321); ray / hit are SoA blocks of N lanes."""
    _fields_ = [("valid", C.POINTER(C.c_int)), ("geometryUserPtr", C.c_void_p), ("context", C.POINTER(RayQueryContext)),
                ("ray", C.POINTER(C.c_uint)), ("hit", C.POINTER(C.c_uint)), ("N", C.c_uint)]


FILTER_FUNCTION = C.CFUNCTYPE(None, C.POINTER(FilterFunctionNArguments))
RTC_RAY_QUERY_FLAG_INVOKE_ARGUMENT_FILTER = 1 << 1


def filter_lane(args, lane):
    """Python view of lane `lane` of a filter callback's arguments: dict of the ray / hit fields (u32 bit patterns for
    ids, floats for the rest), as RTCRayN_* / RTCHitN_* (rtcore_ray.h:187-256) read them."""
    a = args.contents
    n = a.N
    ray = np.ctypeslib.as_array(a.ray, shape=(12 * n,))
    hit = np.ctypeslib.as_array(a.hit, shape=(9 * n,))
    out = {}
    for f, name in enumerate(_RAY_FIELDS):
        w = ray[f * n + lane]
        out[name] = int(w) if name in ("mask", "id", "flags") else float(np.uint32(w).view(np.float32))
    for f, name in enumerate(_HIT_FIELDS):
        w = hit[f * n + lane]
        out[name] = int(w) if name in ("primID", "geomID", "instID", "instPrimID") else float(np.uint32(w).view(np.float32))
    return out


class InterpolateArguments(C.Structure):
    """RTCInterpolateArguments (rtcore_geometry.h:284-299)."""
    _fields_ = [("geometry", C.c_void_p), ("primID", C.c_uint), ("u", C.c_float), ("v", C.c_float), ("bufferType", C.c_int), ("bufferSlot", C.c_uint),
                ("P", C.c_void_p), ("dPdu", C.c_void_p), ("dPdv", C.c_void_p), ("ddPdudu", C.c_void_p), ("ddPdvdv", C.c_void_p), ("ddPdudv", C.c_void_p),
                ("valueCount", C.c_uint)]


class RTCBounds(C.Structure):
    _fields_ = [(n, C.c_float) for n in
                ("lower_x", "lower_y", "lower_z", "align0", "upper_x", "upper_y", "upper_z", "align1")]


class SceneStats(C.Structure):
    _fields_ = [("num_triangles", C.c_ulonglong), ("num_nodes", C.c_ulonglong), ("node_bytes", C.c_ulonglong),
                ("tri_bytes", C.c_ulonglong), ("build_ms", C.c_double), ("sah_cost", C.c_double),
                ("trav_rays", C.c_ulonglong), ("trav_nodes", C.c_ulonglong), ("trav_tris", C.c_ulonglong),
                ("builder", C.c_uint), ("max_depth", C.c_uint)]


class SceneLayout(C.Structure):
    _fields_ = [(n, C.c_uint) for n in ("num_nodes", "num_records", "num_descs", "num_levels", "num_subs", "top_nodes", "max_depth",
                                        "general", "robust", "builder")]


DESC_DTYPE = np.dtype([("geomID", "<u4"), ("instID", "<u4"), ("kind", "<u4"), ("first", "<u4"), ("count", "<u4"), ("is_quad", "<u4"),
                       ("tess", "<u4"), ("basis", "<u4"), ("hermite", "<u4"), ("xfm", "<f4", (12,))])   # RTCB200DescInfo


def _ptr(a):
    return C.c_void_p(a.ctypes.data) if isinstance(a, np.ndarray) else C.c_void_p(a)


class RTCLib:
    """One loaded Embree-4-API library.  `is_b200` is True when the rtcb200* extension is exported."""

    _SIGS = {
        "rtcNewDevice": (C.c_void_p, [C.c_char_p]),
        "rtcRetainDevice": (None, [C.c_void_p]),
        "rtcReleaseDevice": (None, [C.c_void_p]),
        "rtcGetDeviceProperty": (C.c_ssize_t, [C.c_void_p, C.c_int]),
        "rtcSetDeviceProperty": (None, [C.c_void_p, C.c_int, C.c_ssize_t]),
        "rtcGetErrorString": (C.c_char_p, [C.c_int]),
        "rtcGetDeviceError": (C.c_int, [C.c_void_p]),
        "rtcGetDeviceLastErrorMessage": (C.c_char_p, [C.c_void_p]),
        "rtcSetDeviceErrorFunction": (None, [C.c_void_p, C.c_void_p, C.c_void_p]),
        "rtcSetDeviceMemoryMonitorFunction": (None, [C.c_void_p, C.c_void_p, C.c_void_p]),
        "rtcNewBuffer": (C.c_void_p, [C.c_void_p, C.c_size_t]),
        "rtcNewSharedBuffer": (C.c_void_p, [C.c_void_p, C.c_void_p, C.c_size_t]),
        "rtcGetBufferData": (C.c_void_p, [C.c_void_p]),
        "rtcRetainBuffer": (None, [C.c_void_p]),
        "rtcReleaseBuffer": (None, [C.c_void_p]),
        "rtcNewGeometry": (C.c_void_p, [C.c_void_p, C.c_int]),
        "rtcRetainGeometry": (None, [C.c_void_p]),
        "rtcReleaseGeometry": (None, [C.c_void_p]),
        "rtcCommitGeometry": (None, [C.c_void_p]),
        "rtcEnableGeometry": (None, [C.c_void_p]),
        "rtcDisableGeometry": (None, [C.c_void_p]),
        "rtcSetGeometryMask": (None, [C.c_void_p, C.c_uint]),
        "rtcSetGeometryBuildQuality": (None, [C.c_void_p, C.c_int]),
        "rtcSetGeometryBuffer": (None, [C.c_void_p, C.c_int, C.c_uint, C.c_int, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t]),
        "rtcSetSharedGeometryBuffer": (None, [C.c_void_p, C.c_int, C.c_uint, C.c_int, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t]),
        "rtcSetNewGeometryBuffer": (C.c_void_p, [C.c_void_p, C.c_int, C.c_uint, C.c_int, C.c_size_t, C.c_size_t]),
        "rtcGetGeometryBufferData": (C.c_void_p, [C.c_void_p, C.c_int, C.c_uint]),
        "rtcUpdateGeometryBuffer": (None, [C.c_void_p, C.c_int, C.c_uint]),
        "rtcSetGeometryTessellationRate": (None, [C.c_void_p, C.c_float]),
        "rtcInterpolate": (None, [C.c_void_p]),
        "rtcSetGeometryUserData": (None, [C.c_void_p, C.c_void_p]),
        "rtcGetGeometryUserData": (C.c_void_p, [C.c_void_p]),
        "rtcSetGeometryIntersectFilterFunction": (None, [C.c_void_p, C.c_void_p]),
        "rtcSetGeometryOccludedFilterFunction": (None, [C.c_void_p, C.c_void_p]),
        "rtcSetGeometryEnableFilterFunctionFromArguments": (None, [C.c_void_p, C.c_bool]),
        "rtcSetGeometryInstancedScene": (None, [C.c_void_p, C.c_void_p]),
        "rtcSetGeometryTransform": (None, [C.c_void_p, C.c_uint, C.c_int, C.c_void_p]),
        "rtcGetGeometryTransform": (None, [C.c_void_p, C.c_float, C.c_int, C.c_void_p]),
        "rtcNewScene": (C.c_void_p, [C.c_void_p]),
        "rtcGetSceneDevice": (C.c_void_p, [C.c_void_p]),
        "rtcRetainScene": (None, [C.c_void_p]),
        "rtcReleaseScene": (None, [C.c_void_p]),
        "rtcAttachGeometry": (C.c_uint, [C.c_void_p, C.c_void_p]),
        "rtcAttachGeometryByID": (None, [C.c_void_p, C.c_void_p, C.c_uint]),
        "rtcDetachGeometry": (None, [C.c_void_p, C.c_uint]),
        "rtcGetGeometry": (C.c_void_p, [C.c_void_p, C.c_uint]),
        "rtcCommitScene": (None, [C.c_void_p]),
        "rtcJoinCommitScene": (None, [C.c_void_p]),
        "rtcSetSceneBuildQuality": (None, [C.c_void_p, C.c_int]),
        "rtcSetSceneFlags": (None, [C.c_void_p, C.c_int]),
        "rtcGetSceneFlags": (C.c_int, [C.c_void_p]),
        "rtcGetSceneBounds": (None, [C.c_void_p, C.c_void_p]),
        "rtcIntersect1": (None, [C.c_void_p, C.c_void_p, C.c_void_p]),
        "rtcIntersect4": (None, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
        "rtcIntersect8": (None, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
        "rtcIntersect16": (None, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
        "rtcOccluded1": (None, [C.c_void_p, C.c_void_p, C.c_void_p]),
        "rtcOccluded4": (None, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
        "rtcOccluded8": (None, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
        "rtcOccluded16": (None, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    }
    _EXT_SIGS = {
        "rtcb200Intersect1M": (None, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
        "rtcb200Occluded1M": (None, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
        "rtcb200IntersectNM": (None, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint, C.c_size_t, C.c_void_p]),
        "rtcb200OccludedNM": (None, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint, C.c_size_t, C.c_void_p]),
        "rtcb200Intersect1MDevice": (None, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
        "rtcb200Intersect1MGatherDevice": (None, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]),
        "rtcb200PeerAlloc": (C.c_void_p, [C.c_void_p, C.c_size_t]),
        "rtcb200PeerFree": (None, [C.c_void_p, C.c_void_p]),
        "rtcb200PeerExport": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
        "rtcb200PeerImport": (C.c_void_p, [C.c_void_p, C.c_void_p]),
        "rtcb200PeerClose": (None, [C.c_void_p, C.c_void_p]),
        "rtcb200PeerCopy": (None, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
        "rtcb200Occluded1MDevice": (None, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
        "rtcb200IntersectNMDevice": (None, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint, C.c_size_t, C.c_void_p, C.c_void_p]),
        "rtcb200OccludedNMDevice": (None, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint, C.c_size_t, C.c_void_p, C.c_void_p]),
        "rtcb200GetSceneStats": (None, [C.c_void_p, C.c_void_p]),
        "rtcb200SetSceneStatCounters": (None, [C.c_void_p, C.c_int]),
        "rtcb200ResetSceneStatCounters": (None, [C.c_void_p]),
        "rtcb200GetLaunchCount": (C.c_ulonglong, []),
        "rtcb200SetTuning": (C.c_int, [C.c_char_p, C.c_int]),
        "rtcb200GetLastTraceMs": (C.c_double, [C.c_void_p]),
        "rtcb200GetSceneLayout": (None, [C.c_void_p, C.c_void_p]),
        "rtcb200CopySceneArrays": (None, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    }

    def __init__(self, path):
        if not os.path.exists(path):
            raise FileNotFoundError(f"rtc library not found: {path}")
        self.path = path
        self.dll = C.CDLL(path, mode=C.RTLD_LOCAL)
        for name, (res, args) in self._SIGS.items():
            fn = getattr(self.dll, name)
            fn.restype, fn.argtypes = res, args
            setattr(self, name, fn)
        self.is_b200 = hasattr(self.dll, "rtcb200Intersect1M")
        if self.is_b200:
            for name, (res, args) in self._EXT_SIGS.items():
                fn = getattr(self.dll, name)
                fn.restype, fn.argtypes = res, args
                setattr(self, name, fn)

    # ---- conveniences mirroring what every reference test does ---------------------------------
    def new_device(self, config=None):
        d = self.rtcNewDevice(config.encode() if config else None)
        if not d:
            msg = self.rtcGetDeviceLastErrorMessage(None)
            raise RuntimeError(f"rtcNewDevice failed: {msg.decode() if msg else '?'}")
        return d

    def check(self, device):
        e = self.rtcGetDeviceError(device)
        if e != RTC_ERROR_NONE:
            raise RuntimeError(f"rtc error {self.rtcGetErrorString(e).decode()}")

    def add_triangle_mesh(self, device, scene, vertices, indices, mask=None, quality=None, geom_id=None):
        """rtcNewGeometry + shared vertex/index buffers + commit + attach (tutorials/minimal/minimal.cpp:90-131).
        The arrays must stay alive; the vertex array is padded to 16 B as README.md:4830 requires."""
        v = np.ascontiguousarray(vertices, np.float32).reshape(-1, 3)
        vpad = np.zeros(v.size + 4, np.float32)
        vpad[:v.size] = v.reshape(-1)
        idx = np.ascontiguousarray(indices, np.uint32).reshape(-1, 3)
        g = self.rtcNewGeometry(device, RTC_GEOMETRY_TYPE_TRIANGLE)
        self.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, _ptr(vpad), 0, 12, v.shape[0])
        self.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT3, _ptr(idx), 0, 12, idx.shape[0])
        if mask is not None:
            self.rtcSetGeometryMask(g, mask)
        if quality is not None:
            self.rtcSetGeometryBuildQuality(g, quality)
        self.rtcCommitGeometry(g)
        if geom_id is None:
            gid = self.rtcAttachGeometry(scene, g)
        else:
            self.rtcAttachGeometryByID(scene, g, geom_id)
            gid = geom_id
        self.rtcReleaseGeometry(g)
        return gid, (vpad, idx)

    def add_round_linear_curves(self, device, scene, vertices4, indices, flags=None, mask=None, geom_id=None, flat=False):
        """RTC_GEOMETRY_TYPE_ROUND_LINEAR_CURVE (flat=True: RTC_GEOMETRY_TYPE_FLAT_LINEAR_CURVE) with shared FLOAT4 (xyz, radius)
        vertex / UINT first-vertex index buffers and an optional UCHAR neighbour-flags buffer (tutorials/hair_geometry,
        curve_geometry).  The arrays must stay alive."""
        v = np.ascontiguousarray(vertices4, np.float32).reshape(-1, 4)
        idx = np.ascontiguousarray(indices, np.uint32).reshape(-1)
        g = self.rtcNewGeometry(device, RTC_GEOMETRY_TYPE_FLAT_LINEAR_CURVE if flat else RTC_GEOMETRY_TYPE_ROUND_LINEAR_CURVE)
        self.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT4, _ptr(v), 0, 16, v.shape[0])
        self.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT, _ptr(idx), 0, 4, idx.shape[0])
        keep = [v, idx]
        if flags is not None:
            f = np.ascontiguousarray(flags, np.uint8).reshape(-1)
            self.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_FLAGS, 0, RTC_FORMAT_UCHAR, _ptr(f), 0, 1, f.shape[0])
            keep.append(f)
        if mask is not None:
            self.rtcSetGeometryMask(g, mask)
        self.rtcCommitGeometry(g)
        if geom_id is None:
            gid = self.rtcAttachGeometry(scene, g)
        else:
            self.rtcAttachGeometryByID(scene, g, geom_id)
            gid = geom_id
        self.rtcReleaseGeometry(g)
        return gid, tuple(keep)

    def add_flat_cubic_curves(self, device, scene, vertices4, indices, basis="bezier", tess=None, tangents=None, mask=None, geom_id=None, round=False):
        """RTC_GEOMETRY_TYPE_FLAT_{BEZIER,BSPLINE,CATMULL_ROM,HERMITE}_CURVE: shared FLOAT4 control vertices (xyz, radius), UINT index
        of each curve's first control vertex, FLOAT4 tangents for 'hermite', optional tessellation rate (tutorials/curve_geometry,
        hair_geometry).  The arrays must stay alive."""
        v = np.ascontiguousarray(vertices4, np.float32).reshape(-1, 4)
        idx = np.ascontiguousarray(indices, np.uint32).reshape(-1)
        g = self.rtcNewGeometry(device, (ROUND_CUBIC_TYPES if round else FLAT_CUBIC_TYPES)[basis])   # round=True: RTC_GEOMETRY_TYPE_ROUND_*_CURVE
        self.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT4, _ptr(v), 0, 16, v.shape[0])
        self.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT, _ptr(idx), 0, 4, idx.shape[0])
        keep = [v, idx]
        if basis == "hermite":
            tg = np.ascontiguousarray(tangents, np.float32).reshape(-1, 4)
            self.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_TANGENT, 0, RTC_FORMAT_FLOAT4, _ptr(tg), 0, 16, tg.shape[0])
            keep.append(tg)
        if tess is not None:
            self.rtcSetGeometryTessellationRate(g, float(tess))
        if mask is not None:
            self.rtcSetGeometryMask(g, mask)
        self.rtcCommitGeometry(g)
        if geom_id is None:
            gid = self.rtcAttachGeometry(scene, g)
        else:
            self.rtcAttachGeometryByID(scene, g, geom_id)
            gid = geom_id
        self.rtcReleaseGeometry(g)
        return gid, keep

    def add_points(self, device, scene, vertices4, kind="sphere", normals=None, mask=None, geom_id=None):
        """RTC_GEOMETRY_TYPE_SPHERE_POINT / _DISC_POINT / _ORIENTED_DISC_POINT: shared FLOAT4 vertices (centre, radius), one
        primitive per vertex; 'oriented_disc' adds FLOAT3 normals (tutorials/point_geometry).  The arrays must stay alive."""
        v = np.ascontiguousarray(vertices4, np.float32).reshape(-1, 4)
        g = self.rtcNewGeometry(device, POINT_TYPES[kind])
        self.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT4, _ptr(v), 0, 16, v.shape[0])
        keep = [v]
        if kind == "oriented_disc":
            n = np.ascontiguousarray(normals, np.float32).reshape(-1, 3)
            npad = np.zeros(n.size + 4, np.float32)
            npad[:n.size] = n.reshape(-1)
            self.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_NORMAL, 0, RTC_FORMAT_FLOAT3, _ptr(npad), 0, 12, n.shape[0])
            keep.append(npad)
        if mask is not None:
            self.rtcSetGeometryMask(g, mask)
        self.rtcCommitGeometry(g)
        if geom_id is None:
            gid = self.rtcAttachGeometry(scene, g)
        else:
            self.rtcAttachGeometryByID(scene, g, geom_id)
            gid = geom_id
        self.rtcReleaseGeometry(g)
        return gid, keep

    def add_quad_mesh(self, device, scene, vertices, indices, mask=None, geom_id=None):
        """RTC_GEOMETRY_TYPE_QUAD with shared FLOAT3 vertex / UINT4 index buffers (quad (v0,v1,v2,v3); a triangle is a
        quad with v2 == v3).  The arrays must stay alive."""
        v = np.ascontiguousarray(vertices, np.float32).reshape(-1, 3)
        vpad = np.zeros(v.size + 4, np.float32)
        vpad[:v.size] = v.reshape(-1)
        idx = np.ascontiguousarray(indices, np.uint32).reshape(-1, 4)
        g = self.rtcNewGeometry(device, RTC_GEOMETRY_TYPE_QUAD)
        self.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, _ptr(vpad), 0, 12, v.shape[0])
        self.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT4, _ptr(idx), 0, 16, idx.shape[0])
        if mask is not None:
            self.rtcSetGeometryMask(g, mask)
        self.rtcCommitGeometry(g)
        if geom_id is None:
            gid = self.rtcAttachGeometry(scene, g)
        else:
            self.rtcAttachGeometryByID(scene, g, geom_id)
            gid = geom_id
        self.rtcReleaseGeometry(g)
        return gid, (vpad, idx)

    def add_instance(self, device, scene, child_scene, xfm, mask=None, geom_id=None, fmt=RTC_FORMAT_FLOAT3X4_COLUMN_MAJOR):
        """rtcNewGeometry(INSTANCE) + instanced scene + transform + commit + attach (tutorials/instanced_geometry).
        `xfm`: 12 floats, column-major 3x4 (vx | vy | vz | p) unless `fmt` says otherwise."""
        m = np.ascontiguousarray(xfm, np.float32).reshape(-1)
        g = self.rtcNewGeometry(device, RTC_GEOMETRY_TYPE_INSTANCE)
        self.rtcSetGeometryInstancedScene(g, child_scene)
        self.rtcSetGeometryTransform(g, 0, fmt, _ptr(m))
        if mask is not None:
            self.rtcSetGeometryMask(g, mask)
        self.rtcCommitGeometry(g)
        if geom_id is None:
            gid = self.rtcAttachGeometry(scene, g)
        else:
            self.rtcAttachGeometryByID(scene, g, geom_id)
            gid = geom_id
        self.rtcReleaseGeometry(g)
        return gid

    def args(self, coherent=False, filter=None, invoke_argument_filter=False, context=None):
        """RTCIntersectArguments / RTCOccludedArguments (same layout).  `filter`: a FILTER_FUNCTION instance (keep it
        alive); `context`: a RayQueryContext (or a structure that starts with one)."""
        a = _IntersectArguments()
        a.flags = (RTC_RAY_QUERY_FLAG_COHERENT if coherent else RTC_RAY_QUERY_FLAG_INCOHERENT) | \
                  (RTC_RAY_QUERY_FLAG_INVOKE_ARGUMENT_FILTER if invoke_argument_filter else 0)
        a.feature_mask = RTC_FEATURE_FLAG_ALL
        a.context = C.cast(C.pointer(context), C.c_void_p) if context is not None else None
        a.filter = C.cast(filter, C.c_void_p) if filter is not None else None
        a.intersect = None
        return a

    # "IntersectWithMode": feed the same RTCRayHit[] through any entry point -------------------------
    def intersect(self, scene, rayhits, mode="1", coherent=False, args=None):
        """mode: '1' (loop of rtcIntersect1), '4'/'8'/'16' (loop of packets), '1M'/'4M'/'8M'/'16M' (batched ext)."""
        a = args if args is not None else self.args(coherent)
        n = len(rayhits)
        if mode == "1":
            base, st = rayhits.ctypes.data, rayhits.dtype.itemsize
            for i in range(n):
                self.rtcIntersect1(scene, C.c_void_p(base + i * st), C.byref(a))
            return rayhits
        if mode == "1M":
            self.rtcb200Intersect1M(scene, _ptr(rayhits), n, C.byref(a))
            return rayhits
        K = int(mode.rstrip("M"))
        p, valid = to_packets(rayhits, K)
        if mode.endswith("M"):
            self.rtcb200IntersectNM(_ptr(valid), scene, _ptr(p), K, len(p), C.byref(a))
        else:
            fn = getattr(self, f"rtcIntersect{K}")
            for i in range(len(p)):
                fn(C.c_void_p(valid.ctypes.data + 4 * K * i), scene, C.c_void_p(p.ctypes.data + p.dtype.itemsize * i), C.byref(a))
        rayhits[:] = from_packets(p, n)
        return rayhits

    def occluded(self, scene, rays, mode="1", coherent=False, args=None):
        a = args if args is not None else self.args(coherent)
        n = len(rays)
        if mode == "1":
            base, st = rays.ctypes.data, rays.dtype.itemsize
            for i in range(n):
                self.rtcOccluded1(scene, C.c_void_p(base + i * st), C.byref(a))
            return rays
        if mode == "1M":
            self.rtcb200Occluded1M(scene, _ptr(rays), n, C.byref(a))
            return rays
        K = int(mode.rstrip("M"))
        p, valid = to_packets(rays, K, hit=False)
        if mode.endswith("M"):
            self.rtcb200OccludedNM(_ptr(valid), scene, _ptr(p), K, len(p), C.byref(a))
        else:
            fn = getattr(self, f"rtcOccluded{K}")
            for i in range(len(p)):
                fn(C.c_void_p(valid.ctypes.data + 4 * K * i), scene, C.c_void_p(p.ctypes.data + p.dtype.itemsize * i), C.byref(a))
        rays[:] = from_packets(p, n, hit=False)
        return rays

    def scene_stats(self, scene):
        s = SceneStats()
        self.rtcb200GetSceneStats(scene, C.byref(s))
        return s

    def scene_arrays(self, scene):
        """Copy of a committed scene's acceleration structure (rtcb200CopySceneArrays), for inspection: dict of the layout fields
        and nodes (uint32 [num_nodes, 24]), records (uint32 [num_records, 12]), descs (DESC_DTYPE), levels, subs (uint32 [num_subs, 4])."""
        lay = SceneLayout()
        self.rtcb200GetSceneLayout(scene, C.byref(lay))
        out = {n: getattr(lay, n) for n, _ in SceneLayout._fields_}
        out["nodes"] = np.zeros((lay.num_nodes, 24), np.uint32)
        out["records"] = np.zeros((lay.num_records, 12), np.uint32)
        out["descs"] = np.zeros(lay.num_descs, DESC_DTYPE)
        out["levels"] = np.zeros(lay.num_levels, np.uint32)
        out["subs"] = np.zeros((lay.num_subs, 4), np.uint32)
        self.rtcb200CopySceneArrays(scene, _ptr(out["nodes"]), _ptr(out["records"]), _ptr(out["descs"]), _ptr(out["levels"]), _ptr(out["subs"]))
        return out
