"""Geometry buffers in GPU memory (rtcb200SetSharedGeometryBufferDevice): every scene here is built twice, once from host views and
once from device views -- CUDA tensors holding the same bytes -- and the two must agree: the same BVH nodes and leaf records (in the
order a build happens to lay them out, see assert_same), byte-equal level boundaries, descriptors (their buffer addresses aside) and
scene bounds, and byte-equal closest-hit and any-hit records of seeded rays.

Covered: every primitive kind at LOW and MEDIUM quality, fast and ROBUST, with a non-zero byte offset and an interleaved stride; scenes
mixing host and device views; an instanced child scene of device views; a DYNAMIC REFIT mesh and a two-level DYNAMIC scene moved in
place by torch; the edit sequences of test_scene_edits replayed with device-resident buffers; the snapshot a commit takes (zeroed and
freed tensors change nothing); that interpolation reads the buffers at its first request after a commit; batched and per-hit
device interpolation; and every refusal of the entry point and its getters, and an empty device view.

Both arms of every comparison derive linear-curve neighbour flags with the same kernel (build.cu curve_flags), so these tests do not
hold that kernel to the reference: the golden curve tests (tests/golden/curves.npz and curves_flat.npz, derived and application
flags) do."""
import ctypes as C

import numpy as np
import pytest

from embree_b200 import scenes
from embree_b200.rtc import (FLAT_CUBIC_TYPES, POINT_TYPES, ROUND_CUBIC_TYPES, RTCBounds, InterpolateArguments, InterpolateNArguments,
                             RTC_BUFFER_TYPE_FLAGS, RTC_BUFFER_TYPE_INDEX, RTC_BUFFER_TYPE_NORMAL, RTC_BUFFER_TYPE_TANGENT,
                             RTC_BUFFER_TYPE_VERTEX, RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, RTC_BUILD_QUALITY_LOW, RTC_BUILD_QUALITY_MEDIUM,
                             RTC_BUILD_QUALITY_REFIT, RTC_ERROR_INVALID_ARGUMENT, RTC_ERROR_INVALID_OPERATION, RTC_ERROR_NONE, RTC_FORMAT_FLOAT,
                             RTC_FORMAT_FLOAT3, RTC_FORMAT_FLOAT3X4_COLUMN_MAJOR, RTC_FORMAT_FLOAT4, RTC_FORMAT_UCHAR, RTC_FORMAT_UINT,
                             RTC_FORMAT_UINT3, RTC_FORMAT_UINT4, RTC_GEOMETRY_TYPE_FLAT_LINEAR_CURVE, RTC_GEOMETRY_TYPE_QUAD,
                             RTC_GEOMETRY_TYPE_ROUND_LINEAR_CURVE, RTC_GEOMETRY_TYPE_TRIANGLE, RTC_SCENE_FLAG_DYNAMIC, RTC_SCENE_FLAG_NONE,
                             RTC_SCENE_FLAG_ROBUST, INTERP_OUTPUTS, _ptr, make_rayhits, rays_of)
from tests import test_scene_edits as edits
from tests.test_device_shading import device_interpolate, devshade  # noqa: F401  (devshade: the fixture of rtcb200Interpolate1)

pytestmark = pytest.mark.gpu
INVALID = 0xFFFFFFFF
FORMAT_BYTES = {RTC_FORMAT_UCHAR: 1, RTC_FORMAT_UINT: 4, RTC_FORMAT_UINT3: 12, RTC_FORMAT_UINT4: 16, RTC_FORMAT_FLOAT: 4,
                RTC_FORMAT_FLOAT + 1: 8, RTC_FORMAT_FLOAT3: 12, RTC_FORMAT_FLOAT4: 16}
GEOM_DESC_BYTES = 216                     # sizeof(rtk::GeomDesc)
GEOM_DESC_ADDRESSES = (0, 8, 72, 96, 104)  # its verts, idx, flags, basis_tab and tangents pointers


# ---- buffers: host or device views of the same bytes ---------------------------------------------------------------------
def pack(rows, offset, stride, seed):
    """`rows` (one item per row) at `offset` + i * `stride` of a byte buffer whose other bytes are seeded noise."""
    rows = np.ascontiguousarray(rows)
    items = rows.reshape(len(rows), -1).view(np.uint8)
    buf = np.random.RandomState(seed).randint(0, 256, offset + len(rows) * stride + 16).astype(np.uint8)
    np.lib.stride_tricks.as_strided(buf[offset:], shape=items.shape, strides=(stride, 1))[:] = items
    return buf


class Buffers:
    """Attaches geometry buffers as host views (numpy) or, `device`, as device views (CUDA tensors of the same bytes, through
    RTCLib.set_device_buffer)."""

    def __init__(self, lib, device):
        self.lib, self.device, self.host, self.geoms, self.by_key = lib, device, [], set(), {}

    def set(self, g, btype, slot, fmt, rows, offset, stride, seed):
        import torch
        buf = pack(rows, offset, stride, seed)
        self.host.append(buf)
        self.by_key[(g, btype, slot)] = buf
        if self.device:
            self.lib.set_device_buffer(g, btype, slot, fmt, torch.from_numpy(buf).cuda(), offset, stride, len(rows))
            self.geoms.add(g)
        else:
            self.lib.rtcSetSharedGeometryBuffer(g, btype, slot, fmt, _ptr(buf), offset, stride, len(rows))

    def tensors(self):
        return [t for (g, _, _), t in self.lib._device_buffers.items() if g in self.geoms]

    def release(self):
        for g in self.geoms:
            self.lib.release_device_buffers(g)
        self.geoms.clear()


# ---- geometry of every kind: a type, its buffers (type, slot, format, rows, offset, stride) and its tessellation rate -------------
def strands(rng, n=40, pts=8, box=2.5):
    p = rng.uniform(-box, box, (n, 1, 3)) + np.cumsum(rng.normal(scale=0.25, size=(n, pts, 3)), 1)
    return np.concatenate([p, rng.uniform(0.02, 0.08, (n, pts, 1))], 2).reshape(-1, 4).astype(np.float32)


def kind_spec(kind, rng):
    f4 = lambda v: (RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT4, v, 16, 32)   # float4 rows interleaved in 32-byte records
    if kind == "triangle":
        v, t = scenes.triangle_sphere(24, rng.uniform(-1, 1, 3), 1.5)
        return dict(type=RTC_GEOMETRY_TYPE_TRIANGLE, bufs=[(RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, v, 8, 20),
                                                          (RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT3, t.astype(np.uint32), 4, 16)])
    if kind == "quad":
        v, q = edits.quad_sphere(16, rng.uniform(-1, 1, 3), 1.5)
        return dict(type=RTC_GEOMETRY_TYPE_QUAD, bufs=[(RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, v.astype(np.float32), 8, 20),
                                                      (RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT4, q.astype(np.uint32), 4, 20)])
    if kind.endswith("linear") or kind.endswith("linear_flags"):
        pts = 8
        v = strands(rng, pts=pts)
        # one index per segment; strand ends and dropped segments leave gaps that the derived neighbour flags must see
        idx = np.array([s * pts + j for s in range(len(v) // pts) for j in range(pts - 1) if rng.rand() > 0.15], np.uint32)
        bufs = [f4(v), (RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT, idx, 4, 8)]
        if kind.endswith("_flags"):
            # the application's flags: a random subset of the neighbours the index buffer has (a flag without a neighbour would send
            # the curve test past the vertex buffer, in the reference too) and noise in the six high bits, which must not count
            right = np.append(idx[1:] == idx[:-1] + 1, False)
            left = np.insert(idx[1:] == idx[:-1] + 1, 0, False)
            fl = (left * 1 | right * 2) & rng.randint(0, 4, len(idx)) | rng.randint(0, 64, len(idx)) << 2
            bufs.append((RTC_BUFFER_TYPE_FLAGS, 0, RTC_FORMAT_UCHAR, fl.astype(np.uint8), 3, 2))
        flat = kind.startswith("flat")
        return dict(type=RTC_GEOMETRY_TYPE_FLAT_LINEAR_CURVE if flat else RTC_GEOMETRY_TYPE_ROUND_LINEAR_CURVE, bufs=bufs)
    if kind.startswith("flat_") or kind.startswith("round_"):
        shape, basis = kind.split("_", 1)
        pts = 8
        v = strands(rng, n=24, pts=pts)
        per = pts - 1 if basis == "hermite" else pts - 3
        idx = np.array([s * pts + j for s in range(len(v) // pts) for j in range(per)], np.uint32)
        bufs = [f4(v), (RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT, idx, 4, 8)]
        if basis == "hermite":
            tg = np.concatenate([rng.normal(scale=0.3, size=(len(v), 3)), np.zeros((len(v), 1))], 1).astype(np.float32)
            bufs.append((RTC_BUFFER_TYPE_TANGENT, 0, RTC_FORMAT_FLOAT4, tg, 16, 48))
        return dict(type=(FLAT_CUBIC_TYPES if shape == "flat" else ROUND_CUBIC_TYPES)[basis], bufs=bufs, tess=6 if shape == "flat" else None)
    v = edits.point_set(rng, n=400, box=2.5)
    bufs = [f4(v)]
    if kind == "oriented_disc":
        n = rng.normal(size=(len(v), 3))
        bufs.append((RTC_BUFFER_TYPE_NORMAL, 0, RTC_FORMAT_FLOAT3, (n / np.linalg.norm(n, axis=1, keepdims=True)).astype(np.float32), 4, 16))
    return dict(type=POINT_TYPES[kind], bufs=bufs)


KINDS = (["triangle", "quad", "round_linear", "flat_linear", "round_linear_flags", "flat_linear_flags"] +
         [f"{s}_{b}" for s in ("flat", "round") for b in ("bezier", "bspline", "catmull_rom", "hermite")] +
         ["sphere", "disc", "oriented_disc"])


def add_geometry(lib, dev, sc, spec, bufs, seed, quality=None, nattr=0):
    g = lib.rtcNewGeometry(dev, spec["type"])
    if nattr:
        lib.dll.rtcSetGeometryVertexAttributeCount(C.c_void_p(g), nattr)
    for k, (btype, slot, fmt, rows, off, stride) in enumerate(spec["bufs"]):
        bufs.set(g, btype, slot, fmt, rows, off, stride, seed * 16 + k)
    if spec.get("tess"):
        lib.rtcSetGeometryTessellationRate(g, float(spec["tess"]))
    if quality is not None:
        lib.rtcSetGeometryBuildQuality(g, quality)
    lib.rtcCommitGeometry(g)
    gid = lib.rtcAttachGeometry(sc, g)
    lib.rtcReleaseGeometry(g)
    return gid


def new_scene(lib, dev, quality=RTC_BUILD_QUALITY_MEDIUM, flags=RTC_SCENE_FLAG_NONE):
    sc = lib.rtcNewScene(dev)
    lib.rtcSetSceneBuildQuality(sc, quality)
    lib.rtcSetSceneFlags(sc, flags)
    return sc


def build(lib, dev, specs, device, quality=RTC_BUILD_QUALITY_MEDIUM, flags=RTC_SCENE_FLAG_NONE):
    """A scene of `specs`, geometry i from device views when device(i); returns (scene, [host Buffers, device Buffers])."""
    sc = new_scene(lib, dev, quality, flags)
    bufs = [Buffers(lib, False), Buffers(lib, True)]
    for i, spec in enumerate(specs):
        add_geometry(lib, dev, sc, spec, bufs[1 if device(i) else 0], seed=i)
    lib.rtcCommitScene(sc)
    lib.check(dev)
    return sc, bufs


# ---- what is compared ----------------------------------------------------------------------------------------------------
def seeded_rays(n, seed, box=4.5):
    rng = np.random.RandomState(seed)
    org = rng.uniform(-box, box, (n, 3))
    return make_rayhits(org, rng.uniform(-2.0, 2.0, (n, 3)) - org)


def trace_device(lib, sc, rh):
    """Closest-hit and any-hit records of `rh` through rtcb200Intersect1MDevice / rtcb200Occluded1MDevice."""
    import torch
    st = torch.cuda.current_stream()
    d = torch.from_numpy(rh.view(np.uint8).copy()).cuda()
    r = torch.from_numpy(rays_of(rh).view(np.uint8).copy()).cuda()
    lib.rtcb200Intersect1MDevice(sc, C.c_void_p(d.data_ptr()), len(rh), C.byref(lib.args()), C.c_void_p(st.cuda_stream))
    lib.rtcb200Occluded1MDevice(sc, C.c_void_p(r.data_ptr()), len(rh), C.byref(lib.args()), C.c_void_p(st.cuda_stream))
    torch.cuda.synchronize()
    return d.cpu().numpy(), r.cpu().numpy()


def masked_descs(lib, dev, sc, n):
    """The scene's device descriptors (rtk::GeomDesc) with their buffer addresses zeroed."""
    t = lib.scene_device_traversable(sc)
    lib.check(dev)
    if not n or not t.descs:
        return b""
    raw = np.zeros(n * GEOM_DESC_BYTES, np.uint8)
    lib.rtcb200PeerCopy(dev, _ptr(raw), C.c_void_p(t.descs), raw.nbytes)
    lib.check(dev)
    raw = raw.reshape(n, GEOM_DESC_BYTES)
    for o in GEOM_DESC_ADDRESSES:
        raw[:, o:o + 8] = 0
    return raw.tobytes()


def state(lib, dev, sc, rh, skip_nodes=0):
    """What is compared of a committed scene; `skip_nodes` leaves out the first nodes."""
    arr = lib.scene_arrays(sc)
    arr["nodes"] = arr["nodes"][skip_nodes:]
    b = RTCBounds()
    lib.rtcGetSceneBounds(sc, C.byref(b))
    hits, occ = trace_device(lib, sc, rh)
    lib.check(dev)
    return dict(nodes=arr["nodes"].tobytes(), records=arr["records"].tobytes(), levels=arr["levels"].tobytes(), descs=arr["descs"].tobytes(),
                geom_descs=masked_descs(lib, dev, sc, arr["num_descs"]), bounds=bytes(b), hits=hits.tobytes(), occluded=occ.tobytes(),
                nhits=int((hits.view(np.uint32).reshape(-1, 24)[:, 18] != INVALID).sum()))


def sorted_rows(b, width, mask=()):
    rows = np.frombuffer(b, np.uint32).reshape(-1, width).copy()
    rows[:, list(mask)] = 0
    return np.sort(rows.view(f"V{4 * width}"), axis=0).tobytes()


NODE_BASES = (4, 5)   # words of a BVH8 node that hold where its children and its leaf records start


def assert_same(want, got, what):
    """Everything `state` took is equal.  The build hands out the node and record slots of each BVH level with atomic counters, so two
    builds of the same primitives -- host views both times, too -- may place the same nodes and records in another order within a
    level: nodes (without the two base indices that order sets) and records are compared as sets of rows; the levels' boundaries, the
    descriptors, the bounds and every traced record are compared byte for byte."""
    bad = []
    for k in want:
        if k == "nodes":
            same = sorted_rows(want[k], 24, NODE_BASES) == sorted_rows(got[k], 24, NODE_BASES)
        elif k == "records":
            same = sorted_rows(want[k], 12) == sorted_rows(got[k], 12)
        else:
            same = want[k] == got[k]
        if not same:
            bad.append(k)
    if "hits" in bad:
        w, g = (np.frombuffer(x["hits"], np.uint32).reshape(-1, 24) for x in (want, got))
        diff = (w != g).any(1)
        bad.append(f"{int(diff.sum())} hit records differ, {int((diff & (w[:, 8] == g[:, 8])).sum())} of them at the same tfar")
    assert not bad, (what, bad)
    assert want["nhits"] > 200, (what, want["nhits"])


# ---- every kind ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("robust", [0, 1])
@pytest.mark.parametrize("quality", [RTC_BUILD_QUALITY_LOW, RTC_BUILD_QUALITY_MEDIUM])
@pytest.mark.parametrize("kind", KINDS)
def test_every_kind_from_device_views_equals_host_views(b200, kind, quality, robust):
    lib, dev = b200
    spec = kind_spec(kind, np.random.RandomState(KINDS.index(kind)))
    rh = seeded_rays(1 << 15, 7)
    flags = RTC_SCENE_FLAG_ROBUST if robust else RTC_SCENE_FLAG_NONE
    out = []
    for device in (False, True):
        sc, bufs = build(lib, dev, [spec], lambda i: device, quality, flags)
        out.append(state(lib, dev, sc, rh))
        lib.rtcReleaseScene(sc)
        bufs[1].release()
    assert_same(out[0], out[1], kind)


def test_scene_mixing_host_and_device_views(b200):
    lib, dev = b200
    rng = np.random.RandomState(3)
    specs = [kind_spec(k, rng) for k in ("triangle", "quad", "round_linear_flags", "flat_hermite", "round_bspline", "sphere", "oriented_disc")]
    rh = seeded_rays(1 << 16, 8)
    out = []
    for device in (lambda i: False, lambda i: i % 2 == 1, lambda i: i % 2 == 0):
        sc, bufs = build(lib, dev, specs, device)
        out.append(state(lib, dev, sc, rh))
        lib.rtcReleaseScene(sc)
        bufs[1].release()
    assert_same(out[0], out[1], "odd geometries on the device")
    assert_same(out[0], out[2], "even geometries on the device")


def rotation(rng):
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    return q


def test_instanced_child_scene_of_device_views(b200):
    lib, dev = b200
    rng = np.random.RandomState(4)
    specs = [kind_spec(k, rng) for k in ("triangle", "round_linear", "flat_bezier", "disc")]
    xr = np.random.RandomState(5)
    xfms = [np.concatenate([(rotation(xr) * xr.uniform(0.3, 0.8)).T.reshape(-1), xr.uniform(-3, 3, 3)]).astype(np.float32) for _ in range(5)]
    rh = seeded_rays(1 << 16, 9, box=6.0)
    out = []
    for device in (False, True):
        child, bufs = build(lib, dev, specs, lambda i: device)
        top = new_scene(lib, dev)
        for x in xfms:
            lib.add_instance(dev, top, child, x, fmt=RTC_FORMAT_FLOAT3X4_COLUMN_MAJOR)
        lib.rtcCommitScene(top)
        lib.check(dev)
        out.append(state(lib, dev, top, rh))
        lib.rtcReleaseScene(top)
        lib.rtcReleaseScene(child)
        bufs[1].release()
    assert_same(out[0], out[1], "instances")


# ---- dynamic scenes: tensors moved in place by torch --------------------------------------------------------------------
def vertex_rows(t, offset, stride, n):
    """The float3 vertices inside a packed device buffer, as a strided float32 view that torch edits in place."""
    import torch
    return t[offset:offset + n * stride].view(n, stride)[:, :12].view(torch.float32)


def test_refit_of_a_device_mesh_moved_in_place(b200):
    import torch
    lib, dev = b200
    v, t = scenes.triangle_sphere(120, (0.3, -0.2, 0.1), 1.8)
    spec = dict(type=RTC_GEOMETRY_TYPE_TRIANGLE, bufs=[(RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, v, 8, 20),
                                                      (RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT3, t.astype(np.uint32), 4, 16)])
    rh = seeded_rays(1 << 16, 10)
    scs, bufs = [], []
    for device in (False, True):
        sc = new_scene(lib, dev, RTC_BUILD_QUALITY_MEDIUM, RTC_SCENE_FLAG_DYNAMIC)
        b = Buffers(lib, device)
        add_geometry(lib, dev, sc, spec, b, seed=0, quality=RTC_BUILD_QUALITY_REFIT)
        lib.rtcCommitScene(sc)
        lib.check(dev)
        scs.append(sc)
        bufs.append(b)
    assert_same(state(lib, dev, scs[0], rh), state(lib, dev, scs[1], rh), "first commit")
    tensor = lib._device_buffers[(lib.rtcGetGeometry(scs[1], 0), RTC_BUFFER_TYPE_VERTEX, 0)]
    for step in range(3):
        vertex_rows(tensor, 8, 20, len(v)).mul_(1.0 + 0.05 * step).add_(0.1 * step - 0.05)   # a torch kernel moves the vertices
        torch.cuda.synchronize()                                                            # complete before the commit
        bufs[0].host[0][:] = tensor.cpu().numpy()                                           # the host mesh gets the same bytes
        for sc in scs:
            g = lib.rtcGetGeometry(sc, 0)
            lib.rtcUpdateGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0)
            lib.rtcCommitGeometry(g)
            lib.rtcCommitScene(sc)
            lib.check(dev)
            assert lib.scene_stats(sc).builder == 2, step
        assert_same(state(lib, dev, scs[0], rh), state(lib, dev, scs[1], rh), f"refit {step}")
    for sc in scs:
        lib.rtcReleaseScene(sc)
    bufs[1].release()


def test_two_level_scene_of_device_meshes(b200):
    import torch
    lib, dev = b200
    rng = np.random.RandomState(12)
    specs = []
    for _ in range(8):
        v, t = scenes.triangle_sphere(int(rng.randint(10, 30)), rng.uniform(-3, 3, 3), rng.uniform(0.4, 1.0))
        specs.append(dict(type=RTC_GEOMETRY_TYPE_TRIANGLE, bufs=[(RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, v, 8, 20),
                                                                (RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT3, t.astype(np.uint32), 4, 16)]))
    rh = seeded_rays(1 << 16, 11)
    scs, bufs = [], []
    for device in (False, True):
        sc, b = build(lib, dev, specs, lambda i: device, RTC_BUILD_QUALITY_MEDIUM, RTC_SCENE_FLAG_DYNAMIC)
        scs.append(sc)
        bufs.append(b)
    assert_same(state(lib, dev, scs[0], rh), state(lib, dev, scs[1], rh), "first commit")
    for step, gid in enumerate((2, 5, 2)):
        n = len(specs[gid]["bufs"][0][3])
        tensor = lib._device_buffers[(lib.rtcGetGeometry(scs[1], gid), RTC_BUFFER_TYPE_VERTEX, 0)]
        vertex_rows(tensor, 8, 20, n).add_(0.2 + 0.1 * step)
        torch.cuda.synchronize()
        bufs[0][0].host[2 * gid][:] = tensor.cpu().numpy()
        for sc in scs:
            g = lib.rtcGetGeometry(sc, gid)
            lib.rtcUpdateGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0)
            lib.rtcCommitGeometry(g)
            lib.rtcCommitScene(sc)
            lib.check(dev)
            assert lib.scene_stats(sc).builder == 3, step
        # the assembly reserves 2 * meshes + 8 nodes for the top level and writes only those it uses; the rest keep whatever their
        # allocation held, so the comparison starts after them (the top level's own nodes are covered by the traced records)
        top = 2 * len(specs) + 8
        assert_same(state(lib, dev, scs[0], rh, top), state(lib, dev, scs[1], rh, top), f"mesh {gid} moved")
    for sc in scs:
        lib.rtcReleaseScene(sc)
    bufs[1][1].release()


class DeviceResident:
    """The library as test_scene_edits' model sees it, with every shared buffer device-resident: rtcSetSharedGeometryBuffer attaches a
    CUDA tensor holding the host bytes instead (same offset, stride and count), and rtcUpdateGeometryBuffer first refreshes that tensor
    from the host memory the model edited."""

    def __init__(self, lib):
        self._lib, self._views = lib, {}

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def rtcSetSharedGeometryBuffer(self, g, btype, slot, fmt, ptr, off, stride, num):
        import torch
        nbytes = off + (num - 1) * stride + FORMAT_BYTES[fmt] if num else 16
        host = np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(ptr.value))
        t = torch.from_numpy(host.copy()).cuda()
        torch.cuda.synchronize()
        self._views[(g, btype, slot)] = (host, t)
        self._lib.set_device_buffer(g, btype, slot, fmt, t, off, stride, num)

    def rtcUpdateGeometryBuffer(self, g, btype, slot):
        import torch
        if (g, btype, slot) in self._views:
            host, t = self._views[(g, btype, slot)]
            t.copy_(torch.from_numpy(host.copy()))
            torch.cuda.synchronize()
        self._lib.rtcUpdateGeometryBuffer(g, btype, slot)

    def release(self):
        for g, _, _ in self._views:
            self._lib.release_device_buffers(g)
        self._views.clear()


@pytest.mark.parametrize("profile", ["two_level", "refit", "mixed"])
def test_scene_edit_sequence_with_device_resident_buffers(b200, profile):
    lib, dev = b200
    seed = edits.SEEDS[profile][0]
    rays = edits.profile_rays(seed, edits.RAY_BOX[profile])
    runs = []
    for L in (lib, DeviceResident(lib)):
        out = []

        def on_commit(k, label, m):
            got = lib.intersect(m.sc, rays.copy(), "1M")
            occ = lib.occluded(m.sc, rays_of(rays), "1M")
            lib.check(dev)
            out.append((label, lib.scene_stats(m.sc).builder, got.tobytes(), occ.tobytes()))
        edits.run_sequence(L, dev, profile, seed, on_commit)
        if L is not lib:
            L.release()
        runs.append(out)
    assert len(runs[0]) == len(runs[1]) == edits.N_COMMITS + 1
    for k, (h, d) in enumerate(zip(*runs)):
        assert h == d, (profile, seed, k, h[0], d[0])


# ---- the snapshot a commit takes -----------------------------------------------------------------------------------------
def test_zeroed_and_freed_tensors_leave_the_committed_scene_unchanged(b200):
    import torch
    lib, dev = b200
    rng = np.random.RandomState(13)
    specs = [kind_spec(k, rng) for k in ("triangle", "quad", "round_linear", "flat_linear_flags", "round_hermite", "flat_catmull_rom", "sphere",
                                         "oriented_disc")]
    rh = seeded_rays(1 << 16, 14)
    sc, bufs = build(lib, dev, specs, lambda i: True)
    before = state(lib, dev, sc, rh)
    ts = bufs[1].tensors()
    assert len(ts) == sum(len(s["bufs"]) for s in specs)
    for t in ts:
        t.zero_()
    torch.cuda.synchronize()
    assert_same(before, state(lib, dev, sc, rh), "tensors zeroed")
    bufs[1].release()
    del ts, t
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    assert_same(before, state(lib, dev, sc, rh), "tensors freed")
    lib.rtcReleaseScene(sc)


# ---- interpolation -------------------------------------------------------------------------------------------------------
def interp_specs(rng):
    specs = [kind_spec(k, rng) for k in ("triangle", "quad", "round_linear", "flat_hermite", "round_bezier")]
    for s in specs:
        n = len(s["bufs"][0][3])
        s["bufs"].append((RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 0, RTC_FORMAT_FLOAT3, rng.normal(size=(n, 3)).astype(np.float32), 12, 28))
    return specs


def build_interp(lib, dev, specs, device):
    sc = new_scene(lib, dev)
    bufs = Buffers(lib, device)
    for i, spec in enumerate(specs):
        add_geometry(lib, dev, sc, spec, bufs, seed=i, nattr=1)
    lib.rtcCommitScene(sc)
    lib.check(dev)
    return sc, bufs


def test_interpolation_of_device_views_equals_host_views(b200, devshade):
    import torch
    lib, dev = b200
    specs = interp_specs(np.random.RandomState(15))
    rh = seeded_rays((1 << 16) + 5, 16)
    built = [build_interp(lib, dev, specs, device) for device in (False, True)]
    hits, _ = trace_device(lib, built[0][0], rh)
    d_hits = torch.from_numpy(hits.copy()).cuda()
    st = torch.cuda.current_stream()
    for bt, vc in ((RTC_BUFFER_TYPE_VERTEX, 3), (RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 3)):
        batched, per_hit = [], []
        for sc, _ in built:
            r = lib.interpolate_hits(sc, d_hits, bt, 0, vc, want=INTERP_OUTPUTS, stream=st)
            torch.cuda.synchronize()
            lib.check(dev)
            batched.append({k: r[k].cpu().numpy().tobytes() for k in INTERP_OUTPUTS})
            o = device_interpolate(lib, dev, devshade, sc, d_hits, bt, 0, vc, st)
            st.synchronize()
            per_hit.append({k: o[k].cpu().numpy().tobytes() for k in INTERP_OUTPUTS})
        assert batched[0] == batched[1], bt
        assert per_hit[0] == per_hit[1], bt
    for sc, b in built:
        lib.rtcReleaseScene(sc)
    built[1][1].release()


def test_interpolation_reads_the_buffers_at_its_first_request_after_a_commit(b200):
    """The commit copies nothing for interpolation: the first batched request copies the buffers as they are then (host and device
    views alike), keeps the copies until the next commit, and a commit after rtcUpdateGeometryBuffer reads the new contents."""
    import torch
    lib, dev = b200
    specs = interp_specs(np.random.RandomState(19))
    built = [build_interp(lib, dev, specs, device) for device in (False, True)]
    hits, _ = trace_device(lib, built[0][0], seeded_rays(1 << 15, 20))
    d_hits = torch.from_numpy(hits.copy()).cuda()
    hit = hits.view(np.uint32).reshape(-1, 24)[:, 18] != INVALID
    st = torch.cuda.current_stream()

    def attrs(edit):
        """edit(host array, device tensor or None) on every geometry's attribute buffer of both scenes"""
        for sc, b in built:
            for gid in range(len(specs)):
                g = lib.rtcGetGeometry(sc, gid)
                key = (g, RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 0)
                edit(b.by_key[key], lib._device_buffers[key] if b.device else None)
        torch.cuda.synchronize()

    def interp():
        out = []
        for sc, _ in built:
            r = lib.interpolate_hits(sc, d_hits, RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 0, 3, want=("P",), stream=st)["P"]
            torch.cuda.synchronize()
            lib.check(dev)
            out.append(r.cpu().numpy())
        assert out[0].view(np.uint32).tobytes() == out[1].view(np.uint32).tobytes()
        return out[0]

    saved = []
    attrs(lambda h, t: saved.append(h.copy()))
    rows = iter(saved)

    def zero(h, t):
        h.fill(0)
        if t is not None:
            t.zero_()

    def restore(h, t):
        h[:] = next(rows)
        if t is not None:
            t.copy_(torch.from_numpy(h))

    attrs(zero)                                       # after the commit, before the first request
    assert (interp()[:, hit] == 0).all()
    attrs(restore)
    assert (interp()[:, hit] == 0).all()              # the table of this commit is kept
    for sc, _ in built:
        for gid in range(len(specs)):
            g = lib.rtcGetGeometry(sc, gid)
            lib.rtcUpdateGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 0)
            lib.rtcCommitGeometry(g)
        lib.rtcCommitScene(sc)
        lib.check(dev)
    assert (interp()[:, hit] != 0).any()              # the next commit's table: the restored values
    for sc, b in built:
        lib.rtcReleaseScene(sc)
    built[1][1].release()


def test_host_interpolate_refuses_device_views(b200):
    lib, dev = b200
    specs = interp_specs(np.random.RandomState(17))
    for device in (False, True):
        sc, bufs = build_interp(lib, dev, specs, device)
        for gid in range(len(specs)):
            g = lib.rtcGetGeometry(sc, gid)
            for bt in (RTC_BUFFER_TYPE_VERTEX, RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE):
                P = np.full(3, 7.0, np.float32)
                a = InterpolateArguments(geometry=g, primID=0, u=0.25, v=0.25, bufferType=bt, bufferSlot=0, P=P.ctypes.data, valueCount=3)
                lib.rtcInterpolate(C.byref(a))
                N = 4
                PN = np.full(3 * N, 7.0, np.float32)
                ids, uv = np.zeros(N, np.uint32), np.full(N, 0.25, np.float32)
                an = InterpolateNArguments(geometry=g, primIDs=ids.ctypes.data, u=uv.ctypes.data, v=uv.ctypes.data, N=N, bufferType=bt,
                                           bufferSlot=0, P=PN.ctypes.data, valueCount=3)
                lib.rtcInterpolateN(C.byref(an))
                err = lib.rtcGetDeviceError(dev)
                if device:
                    assert err == RTC_ERROR_INVALID_OPERATION and (P == 7.0).all() and (PN == 7.0).all(), (gid, bt)
                else:
                    assert err == RTC_ERROR_NONE and not (P == 7.0).all() and not (PN == 7.0).all(), (gid, bt)
        lib.rtcReleaseScene(sc)
        bufs.release()


# ---- refusals and getters ------------------------------------------------------------------------------------------------
def test_refusals_and_getters(b200):
    import torch
    lib, dev = b200
    assert lib.rtcGetDeviceError(dev) == RTC_ERROR_NONE
    v = np.zeros((8, 4), np.float32)
    g = lib.rtcNewGeometry(dev, RTC_GEOMETRY_TYPE_TRIANGLE)
    setd = lib.rtcb200SetSharedGeometryBufferDevice

    def attached():
        p = lib.rtcGetGeometryBufferDataDevice(g, RTC_BUFFER_TYPE_VERTEX, 0)
        assert lib.rtcGetDeviceError(dev) == RTC_ERROR_NONE
        return p

    setd(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, _ptr(v), 0, 16, 8)            # pageable host memory
    assert lib.rtcGetDeviceError(dev) == RTC_ERROR_INVALID_ARGUMENT and attached() is None
    pinned = torch.zeros(32, dtype=torch.float32).pin_memory()
    setd(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, C.c_void_p(pinned.data_ptr()), 0, 16, 8)   # pinned host memory
    assert lib.rtcGetDeviceError(dev) == RTC_ERROR_INVALID_ARGUMENT and attached() is None
    setd(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, None, 0, 16, 8)                # NULL with items
    assert lib.rtcGetDeviceError(dev) == RTC_ERROR_INVALID_ARGUMENT and attached() is None

    d = torch.zeros(64, dtype=torch.float32, device="cuda")
    hv = np.zeros(64, np.float32)
    for off, stride in ((2, 16), (0, 14), (4, 12)):     # misaligned offset, misaligned stride, then a good view
        lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, _ptr(hv), off, stride, 8)
        host_err = lib.rtcGetDeviceError(dev)
        setd(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, C.c_void_p(d.data_ptr()), off, stride, 8)
        assert lib.rtcGetDeviceError(dev) == host_err, (off, stride)
        assert (host_err == RTC_ERROR_NONE) == ((off, stride) == (4, 12)), (off, stride, host_err)
    assert attached() == d.data_ptr() + 4
    assert lib.rtcGetGeometryBufferData(g, RTC_BUFFER_TYPE_VERTEX, 0) is None
    assert lib.rtcGetDeviceError(dev) == RTC_ERROR_INVALID_OPERATION
    lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, _ptr(hv), 4, 12, 8)   # a host view again
    assert lib.rtcGetGeometryBufferData(g, RTC_BUFFER_TYPE_VERTEX, 0) == hv.ctypes.data + 4 == attached()

    # set_device_buffer keeps the tensor of the attached view: a refused call leaves the one attached before referenced
    lib.set_device_buffer(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, d, 4, 12, 8)
    assert lib.rtcGetDeviceError(dev) == RTC_ERROR_NONE and lib._device_buffers[(g, RTC_BUFFER_TYPE_VERTEX, 0)] is d
    other = torch.zeros(64, dtype=torch.float32, device="cuda")
    lib.set_device_buffer(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, other, 2, 12, 8)
    assert lib.rtcGetDeviceError(dev) == RTC_ERROR_INVALID_OPERATION
    assert lib._device_buffers[(g, RTC_BUFFER_TYPE_VERTEX, 0)] is d and attached() == d.data_ptr() + 4
    lib.release_device_buffers(g)
    lib.rtcReleaseGeometry(g)


def test_empty_device_view(b200):
    """NULL with no items attaches an empty view: no address from either getter, and a commit copies nothing from it."""
    import torch
    lib, dev = b200
    sc = new_scene(lib, dev)
    g = lib.rtcNewGeometry(dev, RTC_GEOMETRY_TYPE_ROUND_LINEAR_CURVE)
    lib.rtcb200SetSharedGeometryBufferDevice(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT4, None, 16, 16, 0)
    assert lib.rtcGetDeviceError(dev) == RTC_ERROR_NONE
    assert lib.rtcGetGeometryBufferDataDevice(g, RTC_BUFFER_TYPE_VERTEX, 0) is None
    assert lib.rtcGetDeviceError(dev) == RTC_ERROR_NONE
    assert lib.rtcGetGeometryBufferData(g, RTC_BUFFER_TYPE_VERTEX, 0) is None
    assert lib.rtcGetDeviceError(dev) == RTC_ERROR_INVALID_OPERATION
    idx = torch.zeros(2, dtype=torch.int32, device="cuda")   # two segments over vertices the geometry does not have
    lib.set_device_buffer(g, RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT, idx, 0, 4, 2)
    lib.rtcCommitGeometry(g)
    lib.rtcAttachGeometry(sc, g)
    lib.rtcCommitScene(sc)
    lib.check(dev)
    hits, occ = trace_device(lib, sc, seeded_rays(1024, 21))
    lib.check(dev)
    assert (hits.view(np.uint32).reshape(-1, 24)[:, 18] == INVALID).all()
    lib.rtcReleaseScene(sc)
    lib.rtcReleaseGeometry(g)
    lib.release_device_buffers(g)
