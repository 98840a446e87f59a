"""Scene commits on a CUDA stream (rtcb200CommitSceneWithStream).  Every scene here is committed twice in lockstep: once the
synchronous way (torch.cuda.synchronize(), then rtcCommitScene) and once on a torch stream S without a synchronisation, and the two
must agree: byte-identical traced records and the same BVH nodes and leaf records (as sets of rows, see
test_device_buffers.assert_same).  Where ordering matters, S is first held by one torch.cuda._sleep of about 20 ms, so that a commit
or a reader that does not follow S reads the vertices before the move and shows up as wrong records.

Covered: a refit from device views that returns before S has run; 16 frames of move, commit, trace and interpolation with one
synchronisation; every other reader of a stream-committed scene; every commit path on a stream; refusals (NULL scene, uncommitted
geometry, a capturing stream), releasing a scene right after a stream commit, and the NULL stream."""
import ctypes as C

import numpy as np
import pytest

from embree_b200 import scenes
from embree_b200.rtc import (RAYHIT_DTYPE, RTC_BUFFER_TYPE_INDEX, RTC_BUFFER_TYPE_VERTEX, RTC_BUILD_QUALITY_LOW, RTC_BUILD_QUALITY_MEDIUM,
                             RTC_BUILD_QUALITY_REFIT, RTC_ERROR_INVALID_ARGUMENT, RTC_ERROR_INVALID_OPERATION, RTC_ERROR_NONE,
                             RTC_FORMAT_FLOAT3, RTC_FORMAT_FLOAT3X4_COLUMN_MAJOR, RTC_FORMAT_UINT3, RTC_GEOMETRY_TYPE_TRIANGLE,
                             RTC_SCENE_FLAG_DYNAMIC, RTC_SCENE_FLAG_NONE, RTC_SCENE_FLAG_ROBUST, RTCBounds)
from tests import test_device_buffers as db
from tests.test_device_traversal import devtrace  # noqa: F401  (the fixture of the device-side query launcher)

pytestmark = pytest.mark.gpu
SLEEP_CYCLES = 30_000_000   # about 20 ms at the H100's clocks
INVALID = 0xFFFFFFFF


def torch():
    import torch as t
    return t


# ---- a DYNAMIC scene of one REFIT triangle mesh whose buffers are CUDA tensors --------------------------------------------
class Mesh:
    """A scene of one triangle mesh (device views: float32 [n, 3] vertices, int32 [m, 3] indices)."""

    def __init__(self, lib, dev, num_phi, flags=RTC_SCENE_FLAG_DYNAMIC, quality=RTC_BUILD_QUALITY_REFIT, scene_quality=RTC_BUILD_QUALITY_MEDIUM):
        T = torch()
        v, t = scenes.triangle_sphere(num_phi, (0.1, -0.2, 0.05), 1.5)
        self.lib, self.v = lib, T.from_numpy(np.ascontiguousarray(v, np.float32)).cuda()
        self.idx = T.from_numpy(np.ascontiguousarray(t, np.int32)).cuda()
        self.sc = db.new_scene(lib, dev, scene_quality, flags)
        g = lib.rtcNewGeometry(dev, RTC_GEOMETRY_TYPE_TRIANGLE)
        T.cuda.synchronize()
        lib.set_device_buffer(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, self.v)
        lib.set_device_buffer(g, RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT3, self.idx)
        lib.rtcSetGeometryBuildQuality(g, quality)
        lib.rtcCommitGeometry(g)
        lib.rtcAttachGeometry(self.sc, g)
        lib.rtcReleaseGeometry(g)
        self.g = g
        lib.rtcCommitScene(self.sc)
        lib.check(dev)

    def move(self, step):
        """A torch kernel moves the vertices in place (on the current stream); the geometry is marked updated."""
        self.v.mul_(1.0 + 0.03 * (step + 1)).add_(0.05 * (step + 1))
        self.lib.rtcUpdateGeometryBuffer(self.g, RTC_BUFFER_TYPE_VERTEX, 0)
        self.lib.rtcCommitGeometry(self.g)

    def release(self):
        self.lib.release_device_buffers(self.g)
        self.lib.rtcReleaseScene(self.sc)


def rays(n, seed=3):
    return db.seeded_rays(n, seed, box=3.0)


def on_device(rh):
    """A CUDA tensor holding the records `rh`, complete when this returns (made before a test holds its stream: a device-wide
    synchronisation afterwards would wait for that stream too)."""
    T = torch()
    d = T.from_numpy(rh.view(np.uint8).copy()).cuda()
    T.cuda.synchronize()
    return d


def trace_into(lib, sc, d, stream):
    """rtcb200Intersect1MDevice of the records in tensor `d`, enqueued on `stream`; returns `d`."""
    lib.rtcb200Intersect1MDevice(sc, C.c_void_p(d.data_ptr()), d.numel() // 96, C.byref(lib.args()), C.c_void_p(stream.cuda_stream))
    return d


def sync_trace(lib, sc, rh):
    T = torch()
    out = trace_into(lib, sc, on_device(rh), T.cuda.current_stream()).cpu().numpy().view(RAYHIT_DTYPE)
    T.cuda.synchronize()
    return out


def arrays(lib, sc, skip_nodes=0):
    """The scene's BVH nodes and records as sets of rows (test_device_buffers.assert_same), its descriptors, levels and bounds."""
    a = lib.scene_arrays(sc)
    b = RTCBounds()
    lib.rtcGetSceneBounds(sc, C.byref(b))
    return (db.sorted_rows(a["nodes"][skip_nodes:].tobytes(), 24, db.NODE_BASES), db.sorted_rows(a["records"].tobytes(), 12),
            a["descs"].tobytes(), a["levels"].tobytes(), bytes(b))


def assert_records_equal(want, got, what):
    w, g = (np.asarray(x).view(np.uint32).reshape(-1, 24) for x in (want, got))
    bad = (w != g).any(1)
    assert not bad.any(), (what, int(bad.sum()))
    assert (w[:, 18] != INVALID).sum() > len(w) // 20, what   # enough hits to mean something


def hold(stream):
    """Holds `stream` for about 20 ms: what is enqueued after it runs only then."""
    T = torch()
    with T.cuda.stream(stream):
        T.cuda._sleep(SLEEP_CYCLES)


# ---- 1. a refit returns without waiting -----------------------------------------------------------------------------------
def test_refit_on_a_stream_returns_before_the_stream_ran(b200, capfd):
    T = torch()
    lib, _ = b200
    dev = lib.new_device("verbose=2")
    try:
        ref, m = Mesh(lib, dev, 224), Mesh(lib, dev, 224)   # ~200 k triangles each
        rh = rays(1 << 18)
        before = sync_trace(lib, m.sc, rh)
        ref.move(0)
        T.cuda.synchronize()
        lib.rtcCommitScene(ref.sc)
        lib.check(dev)
        d = on_device(rh)
        S = T.cuda.Stream()
        hold(S)
        with T.cuda.stream(S):
            m.move(0)
        capfd.readouterr()
        lib.commit_on_stream(m.sc, S)
        assert not S.query()                  # the call did not wait for S
        got = trace_into(lib, m.sc, d, S)
        err = capfd.readouterr().err
        lib.check(dev)
        assert "refit" in err and "without a host wait" in err, err
        S.synchronize()
        want = sync_trace(lib, ref.sc, rh)
        assert_records_equal(want, got.cpu().numpy(), "refit on S")
        assert (want.view(np.uint32).reshape(-1, 24) != before.view(np.uint32).reshape(-1, 24)).any()
        assert arrays(lib, ref.sc) == arrays(lib, m.sc)
        assert lib.scene_stats(m.sc).builder == 2
        ref.release()
        m.release()
    finally:
        lib.rtcReleaseDevice(dev)


# ---- 2. frames with one synchronisation ------------------------------------------------------------------------------------
def test_sixteen_frames_with_one_synchronisation(b200):
    T = torch()
    lib, dev = b200
    ref, m = Mesh(lib, dev, 96), Mesh(lib, dev, 96)
    rh = rays(1 << 16, seed=5)
    frames = 16
    want = []
    for f in range(frames):   # the synchronous loop
        ref.move(f)
        T.cuda.synchronize()
        lib.rtcCommitScene(ref.sc)
        hits = trace_into(lib, ref.sc, on_device(rh), T.cuda.current_stream())
        P = lib.interpolate_hits(ref.sc, hits, RTC_BUFFER_TYPE_VERTEX, 0, 3, want=("P",))["P"]
        T.cuda.synchronize()
        want.append((hits.cpu().numpy(), P.cpu().numpy()))
    lib.check(dev)
    S = T.cuda.Stream()
    src = T.from_numpy(rh.view(np.uint8).copy()).cuda()
    bufs = [src.clone() for _ in range(frames)]
    T.cuda.synchronize()
    hold(S)
    got = []
    with T.cuda.stream(S):
        for f in range(frames):
            m.move(f)
            lib.commit_on_stream(m.sc, S)
            trace_into(lib, m.sc, bufs[f], S)
            got.append(lib.interpolate_hits(m.sc, bufs[f], RTC_BUFFER_TYPE_VERTEX, 0, 3, want=("P",), stream=S)["P"])
    T.cuda.synchronize()
    lib.check(dev)
    for f in range(frames):
        assert_records_equal(want[f][0], bufs[f].cpu().numpy(), f"frame {f}")
        w, g = want[f][1], got[f].cpu().numpy()
        assert w.tobytes() == g.tobytes(), f"frame {f}: interpolation"
    assert arrays(lib, ref.sc) == arrays(lib, m.sc)
    ref.release()
    m.release()


# ---- 3. every other reader sees the stream commit ---------------------------------------------------------------------------
CONSUMERS = ["intersect1", "intersect1M", "device_other_stream", "interpolate_hits", "bounds", "stats", "device_query_kernel",
             "parent_commit"]


def read(lib, dev, sc, how, rh, d, devtrace, stream):
    """What the consumer `how` makes of scene `sc` (numpy arrays or bytes); `d`: `rh` on the device, overwritten."""
    T = torch()
    if how == "intersect1":
        return lib.intersect(sc, rh[:512].copy(), mode="1").view(np.uint8)
    if how == "intersect1M":
        return lib.intersect(sc, rh.copy(), mode="1M").view(np.uint8)
    if how == "device_other_stream":
        S2 = T.cuda.Stream()
        trace_into(lib, sc, d, S2)
        S2.synchronize()
        return d.cpu().numpy()
    if how == "interpolate_hits":
        return lib.interpolate_hits(sc, rh, RTC_BUFFER_TYPE_VERTEX, 0, 3, want=("P",))["P"]
    if how == "bounds":
        b = RTCBounds()
        lib.rtcGetSceneBounds(sc, C.byref(b))
        return np.frombuffer(bytes(b), np.uint8)
    if how == "stats":
        s = lib.scene_stats(sc)
        assert s.builder == 2 and s.build_ms > 0, (s.builder, s.build_ms)
        return np.array([s.num_triangles, s.num_nodes, s.builder])
    if how == "device_query_kernel":   # a traversable taken after the commit, the kernel on the commit's stream
        t = lib.scene_device_traversable(sc)
        with T.cuda.stream(stream):
            assert devtrace.devtrace_intersect(C.byref(t), C.c_void_p(d.data_ptr()), len(rh), None, C.c_void_p(stream.cuda_stream)) == 0
        stream.synchronize()
        return d.cpu().numpy()
    assert how == "parent_commit"
    top = db.new_scene(lib, dev)
    lib.add_instance(dev, top, sc, np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0.25, 0, 0], np.float32), fmt=RTC_FORMAT_FLOAT3X4_COLUMN_MAJOR)
    lib.rtcCommitScene(top)
    cur = T.cuda.current_stream()
    trace_into(lib, top, d, cur)
    cur.synchronize()
    lib.rtcReleaseScene(top)
    return d.cpu().numpy()


@pytest.mark.parametrize("how", CONSUMERS)
def test_every_reader_sees_a_stream_commit(b200, devtrace, how):
    T = torch()
    lib, dev = b200
    ref, m = Mesh(lib, dev, 128), Mesh(lib, dev, 128)
    rh = rays(1 << 16, seed=7)
    if how == "interpolate_hits":   # hits of the moved mesh, interpolated by both scenes
        rh = None
    ref.move(0)
    T.cuda.synchronize()
    lib.rtcCommitScene(ref.sc)
    lib.check(dev)
    if rh is None:
        rh = sync_trace(lib, ref.sc, rays(1 << 16, seed=7))
    want = read(lib, dev, ref.sc, how, rh, on_device(rh), devtrace, T.cuda.current_stream())
    d = on_device(rh)
    S = T.cuda.Stream()
    hold(S)
    with T.cuda.stream(S):
        m.move(0)
    lib.commit_on_stream(m.sc, S)
    got = read(lib, dev, m.sc, how, rh, d, devtrace, S)   # no synchronisation in between
    T.cuda.synchronize()
    lib.check(dev)
    assert np.asarray(want).tobytes() == np.asarray(got).tobytes(), how
    ref.release()
    m.release()


# ---- 4. every commit path on a stream ------------------------------------------------------------------------------------
PATHS = ["low", "medium", "robust", "two_level", "flattened", "instance_traversal", "curves_and_points", "host_views"]


class PathScene:
    """One scene of commit path `path` (for instances: the instancing scene) and how a frame edits it."""

    def __init__(self, lib, dev, path):
        self.lib, self.path, self.keep, self.children, self.skip = lib, path, [], [], 0
        rng = np.random.RandomState(PATHS.index(path))
        tri = lambda: db.kind_spec("triangle", rng)
        quality = RTC_BUILD_QUALITY_LOW if path == "low" else RTC_BUILD_QUALITY_MEDIUM
        flags = {"robust": RTC_SCENE_FLAG_ROBUST, "two_level": RTC_SCENE_FLAG_DYNAMIC, "host_views": RTC_SCENE_FLAG_DYNAMIC}.get(path, RTC_SCENE_FLAG_NONE)
        if path == "curves_and_points":
            specs = [db.kind_spec(k, rng) for k in ("triangle", "round_linear", "flat_bezier", "round_catmull_rom", "sphere", "oriented_disc")]
        elif path == "two_level":
            specs = [tri() for _ in range(8)]
            self.skip = 2 * len(specs) + 8   # the top level's reserved nodes (test_device_buffers.test_two_level_scene_of_device_meshes)
        else:
            specs = [tri(), tri()] if path != "host_views" else [tri()]
        self.specs = specs
        device = path != "host_views"
        geom_quality = RTC_BUILD_QUALITY_REFIT if path == "host_views" else None
        target = db.new_scene(lib, dev, quality, flags)
        bufs = db.Buffers(lib, device)
        for i, spec in enumerate(specs):
            db.add_geometry(lib, dev, target, spec, bufs, seed=i, quality=geom_quality)
        self.bufs, self.target, self.nspecs = bufs, target, len(specs)
        lib.rtcCommitScene(target)
        if path in ("flattened", "instance_traversal"):
            self.children.append(target)
            self.sc = db.new_scene(lib, dev)
            xr = np.random.RandomState(11)
            for _ in range(4):
                x = np.concatenate([(db.rotation(xr) * xr.uniform(0.4, 0.8)).T.reshape(-1), xr.uniform(-2, 2, 3)]).astype(np.float32)
                lib.add_instance(dev, self.sc, target, x, fmt=RTC_FORMAT_FLOAT3X4_COLUMN_MAJOR)
            lib.rtcCommitScene(self.sc)
        else:
            self.sc = target
        lib.check(dev)

    def move(self, commit):
        """Moves the vertices of the even geometries (a torch kernel on the current stream, or host memory), then commits the edited
        scene and, for instances, the instancing scene with `commit`."""
        T = torch()
        for gid in range(0, self.nspecs, 2):
            g = self.lib.rtcGetGeometry(self.target, gid)
            key = (g, RTC_BUFFER_TYPE_VERTEX, 0)
            _, _, _, verts, off, stride = self.specs[gid]["bufs"][0]   # the xyz of each vertex row, amid seeded noise
            if self.bufs.device:
                self.lib._device_buffers[key][off:off + len(verts) * stride].view(-1, stride)[:, :12].view(T.float32).add_(0.15)
            else:
                host = self.bufs.by_key[key]
                host[off:off + len(verts) * stride].reshape(-1, stride)[:, :12].view(np.float32)[:] += np.float32(0.15)
            self.lib.rtcUpdateGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0)
            self.lib.rtcCommitGeometry(g)
        for c in self.children:
            commit(c)
        commit(self.sc)

    def release(self):
        self.lib.rtcReleaseScene(self.sc)
        for c in self.children:
            self.lib.rtcReleaseScene(c)
        self.bufs.release()


@pytest.mark.parametrize("path", PATHS)
def test_every_commit_path_on_a_stream(b200, path):
    T = torch()
    lib, dev = b200
    if path == "instance_traversal":
        assert lib.rtcb200SetTuning(b"instance_flatten_max", 0) == 0
    try:
        ref, s = PathScene(lib, dev, path), PathScene(lib, dev, path)
        rh = db.seeded_rays(1 << 16, 13, box=4.5)
        d = on_device(rh)

        def sync_commit(sc):
            T.cuda.synchronize()
            lib.rtcCommitScene(sc)

        ref.move(sync_commit)
        lib.check(dev)
        S = T.cuda.Stream()
        hold(S)
        with T.cuda.stream(S):
            s.move(lambda sc: lib.commit_on_stream(sc, S))
            got = trace_into(lib, s.sc, d, S)
        T.cuda.synchronize()
        lib.check(dev)
        assert_records_equal(sync_trace(lib, ref.sc, rh), got.cpu().numpy(), path)
        assert arrays(lib, ref.sc, ref.skip) == arrays(lib, s.sc, s.skip), path
        if path == "host_views":
            assert lib.scene_stats(s.sc).builder == 2
        ref.release()
        s.release()
    finally:
        if path == "instance_traversal":
            lib.rtcb200SetTuning(b"instance_flatten_max", 2147483647)


# ---- 5. refusals and lifetime --------------------------------------------------------------------------------------------
def test_refusals(b200):
    T = torch()
    lib, dev = b200
    lib.rtcGetDeviceError(None)
    lib.rtcb200CommitSceneWithStream(None, None)
    assert lib.rtcGetDeviceError(None) == RTC_ERROR_INVALID_ARGUMENT
    # an uncommitted geometry: the error rtcCommitScene gives
    m = Mesh(lib, dev, 32)
    m.move(0)
    lib.rtcUpdateGeometryBuffer(m.g, RTC_BUFFER_TYPE_VERTEX, 0)   # modified again, not committed
    lib.rtcCommitScene(m.sc)
    code = lib.rtcGetDeviceError(dev)
    assert code == RTC_ERROR_INVALID_OPERATION
    lib.commit_on_stream(m.sc)
    assert lib.rtcGetDeviceError(dev) == code
    m.release()
    # a capturing stream: refused before anything is enqueued, the scene keeps tracing its last commit
    m = Mesh(lib, dev, 32)
    rh = rays(1 << 14, seed=9)
    before = sync_trace(lib, m.sc, rh)
    m.move(0)
    T.cuda.synchronize()
    x = T.zeros(16, device="cuda")
    g = T.cuda.CUDAGraph()
    with T.cuda.graph(g):
        x.add_(1)
        lib.commit_on_stream(m.sc)
    assert lib.rtcGetDeviceError(dev) == RTC_ERROR_INVALID_OPERATION
    assert_records_equal(before, sync_trace(lib, m.sc, rh), "after the refused capture")
    lib.rtcCommitScene(m.sc)   # the scene commits as usual afterwards
    lib.check(dev)
    assert lib.scene_stats(m.sc).builder == 2
    m.release()


def test_release_right_after_a_stream_commit(b200):
    T = torch()
    lib, dev = b200
    m = Mesh(lib, dev, 128)
    S = T.cuda.Stream()
    hold(S)
    with T.cuda.stream(S):
        m.move(0)
    lib.commit_on_stream(m.sc, S)
    m.release()
    T.cuda.synchronize()
    lib.check(dev)
    assert lib.rtcGetDeviceError(dev) == RTC_ERROR_NONE


def test_null_stream(b200):
    T = torch()
    lib, dev = b200
    ref, m = Mesh(lib, dev, 96), Mesh(lib, dev, 96)
    rh = rays(1 << 16, seed=11)
    for sc_mesh in (ref, m):
        sc_mesh.move(0)
    T.cuda.synchronize()
    lib.rtcCommitScene(ref.sc)
    lib.rtcb200CommitSceneWithStream(m.sc, None)
    lib.check(dev)
    assert_records_equal(sync_trace(lib, ref.sc, rh), sync_trace(lib, m.sc, rh), "NULL stream")
    assert arrays(lib, ref.sc) == arrays(lib, m.sc)
    ref.release()
    m.release()
