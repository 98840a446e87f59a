"""Geometry from GPU memory (rtcb200SetSharedGeometryBufferDevice) against host buffers, on four workloads:

  (a) refit      a 1 M-triangle DYNAMIC REFIT mesh whose vertices a torch kernel moves every frame; one frame is move, update,
                 commit, then 1 Mi rays through rtcb200Intersect1MDevice.  The host arm includes the device-to-host copy of the moved
                 vertices into the shared host buffer that such a caller needs without device buffers.
  (b) rebuild    the same frame with the mesh rebuilt at LOW and at MEDIUM quality instead of refitted
  (c) first      the first commit of the 10 M-triangle createTriangleSphere(1581) (bench.py's scene), vertices and indices already
      commit     where each arm keeps them
  (d) first      the first rtcb200InterpolateHitsDevice (VERTEX, valueCount 3, P + dPdu + dPdv) after that commit, on the hits of
      interp     bench.py's headline stream (64 Mi diffuse bounces): it builds the interpolation table, copying the index and vertex
                 buffers host-to-device or device-to-device

The two arms run alternately: one warm-up each, then --reps repetitions; (a) and (b) time --frames frames per repetition.  CUDA
events on the stream the library commits on and wall clock around them (ending in a synchronise); the report gives median [min, max]
ms per frame / call, the card's name, power limit and max SM clock read in the same call, and whether the two arms' records (hits,
interpolated values) are byte-identical.  Prints one JSON line; writes nothing.

    python scripts/device_buffers_bench.py [--reps R] [--frames F] [--phi-small P] [--phi P] [--rays N]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
import embree_b200  # noqa: E402
from embree_b200 import scenes  # noqa: E402
from embree_b200.rtc import (RTC_BUFFER_TYPE_INDEX, RTC_BUFFER_TYPE_VERTEX, RTC_BUILD_QUALITY_LOW, RTC_BUILD_QUALITY_MEDIUM,  # noqa: E402
                             RTC_BUILD_QUALITY_REFIT, RTC_FORMAT_FLOAT3, RTC_FORMAT_UINT3, RTC_GEOMETRY_TYPE_TRIANGLE, RTC_SCENE_FLAG_DYNAMIC,
                             RTC_SCENE_FLAG_NONE, _ptr, make_rayhits)
from scripts.device_traversal_bench import gpu_info  # noqa: E402


def stat(x):
    return {"ms_median": float(np.median(x)), "ms_range": [float(min(x)), float(max(x))]}


class Mesh:
    """One triangle mesh in a scene of its own, from host views (numpy, padded as README.md:4830 asks) or device views (tensors)."""

    def __init__(self, lib, dev, v, t, device, scene_quality, geom_quality, flags):
        self.lib, self.dev, self.device, self.n = lib, dev, device, len(v)
        self.sc = lib.rtcNewScene(dev)
        lib.rtcSetSceneFlags(self.sc, flags)
        lib.rtcSetSceneBuildQuality(self.sc, scene_quality)
        self.g = lib.rtcNewGeometry(dev, RTC_GEOMETRY_TYPE_TRIANGLE)
        self.vd = torch.from_numpy(np.ascontiguousarray(v, np.float32)).cuda()   # where the caller's kernels move the vertices
        if device:
            self.td = torch.from_numpy(np.ascontiguousarray(t, np.uint32).view(np.int32)).cuda()
            lib.set_device_buffer(self.g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, self.vd, 0, 12, self.n)
            lib.set_device_buffer(self.g, RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT3, self.td, 0, 12, len(t))
        else:
            self.vh = np.zeros(self.n * 3 + 4, np.float32)
            self.vh[:self.n * 3] = np.asarray(v, np.float32).reshape(-1)
            self.vh_t = torch.from_numpy(self.vh[:self.n * 3]).view(self.n, 3)
            self.th = np.ascontiguousarray(t, np.uint32)
            lib.rtcSetSharedGeometryBuffer(self.g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, _ptr(self.vh), 0, 12, self.n)
            lib.rtcSetSharedGeometryBuffer(self.g, RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT3, _ptr(self.th), 0, 12, len(t))
        lib.rtcSetGeometryBuildQuality(self.g, geom_quality)
        lib.rtcCommitGeometry(self.g)
        lib.rtcAttachGeometry(self.sc, self.g)

    def commit(self):
        self.lib.rtcCommitScene(self.sc)

    def moved(self, scale):
        """A frame's vertex edit: a torch kernel moves the vertices; the host arm copies them back to its shared buffer."""
        self.vd.mul_(scale)
        if not self.device:
            self.vh_t.copy_(self.vd)          # device-to-host into pageable memory: returns when the bytes are there
        else:
            torch.cuda.synchronize()          # the commit runs on the library's stream: the writes must be complete
        self.lib.rtcUpdateGeometryBuffer(self.g, RTC_BUFFER_TYPE_VERTEX, 0)
        self.lib.rtcCommitGeometry(self.g)
        self.commit()

    def release(self):
        self.lib.rtcReleaseGeometry(self.g)
        self.lib.rtcReleaseScene(self.sc)
        self.lib.release_device_buffers(self.g)


def timed(fn, stream):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ev[0].record(stream)
    out = fn()
    ev[1].record(stream)
    ev[1].synchronize()
    return ev[0].elapsed_time(ev[1]), (time.perf_counter() - t0) * 1e3, out


def frames(lib, dev, v, t, rays, args, scene_quality, geom_quality, flags, want_builder):
    """(a) / (b): alternating host / device arms of move + update + commit + trace."""
    stream = torch.cuda.current_stream()
    s = C.c_void_p(stream.cuda_stream)
    a = lib.args()
    arms = {name: Mesh(lib, dev, v, t, name == "device", scene_quality, geom_quality, flags) for name in ("host", "device")}
    bufs = {name: torch.empty_like(rays) for name in arms}
    for m in arms.values():
        m.commit()
    lib.check(dev)
    times = {n: {"event": [], "wall": [], "build_ms": []} for n in arms}
    for rep in range(args.reps + 1):
        for name, m in arms.items():
            ev_ms, wall_ms, build = 0.0, 0.0, 0.0
            for f in range(args.frames):
                scale = 1.0005 if f % 2 == 0 else 1.0 / 1.0005

                def frame():
                    m.moved(scale)
                    bufs[name].copy_(rays)
                    lib.rtcb200Intersect1MDevice(m.sc, C.c_void_p(bufs[name].data_ptr()), rays.shape[0], C.byref(a), s)
                e, w, _ = timed(frame, stream)
                st = lib.scene_stats(m.sc)
                assert st.builder == want_builder, (name, st.builder, want_builder)
                ev_ms += e
                wall_ms += w
                build += st.build_ms
            if rep:
                times[name]["event"].append(ev_ms / args.frames)
                times[name]["wall"].append(wall_ms / args.frames)
                times[name]["build_ms"].append(build / args.frames)
    lib.check(dev)
    same = torch.equal(bufs["host"].view(torch.int32), bufs["device"].view(torch.int32))
    hits = int((bufs["device"].view(torch.int32)[:, 18] != -1).sum().item())
    out = {"triangles": len(t), "rays": rays.shape[0], "hits": hits, "records_equal": bool(same)}
    for n in arms:
        out[n] = {"frame_event": stat(times[n]["event"]), "frame_wall": stat(times[n]["wall"]), "device_build_ms": stat(times[n]["build_ms"])}
        arms[n].release()
    out["device_over_host_wall"] = out["device"]["frame_wall"]["ms_median"] / out["host"]["frame_wall"]["ms_median"]
    return out


def first_commit_and_interp(lib, dev, args):
    """(c) and (d): a fresh scene of the 10 M-triangle sphere per repetition and arm; its first commit, then the first (table-building)
    and a second batched interpolation of the headline stream's hits."""
    devt = torch.device("cuda:0")
    stream = torch.cuda.current_stream()
    v, t = bench.make_scene(args.phi)
    v = np.asarray(v, np.float32).reshape(-1, 3)
    t = np.asarray(t, np.uint32).reshape(-1, 3)
    hits = None
    times = {n: {"commit_event": [], "commit_wall": [], "interp_first": [], "interp_second": []} for n in ("host", "device")}
    results = {}
    for rep in range(args.reps + 1):
        for name in ("host", "device"):
            m = Mesh(lib, dev, v, t, name == "device", RTC_BUILD_QUALITY_MEDIUM, RTC_BUILD_QUALITY_MEDIUM, RTC_SCENE_FLAG_NONE)
            torch.cuda.synchronize()
            ce, cw, _ = timed(m.commit, stream)
            lib.check(dev)
            if hits is None:   # the headline stream: primary rays, then 64 Mi diffuse bounces traced through this scene
                prim = scenes.primary_rays(bench.PRIMARY_W, bench.PRIMARY_H, eye=bench.EYE, look=bench.LOOK, device=devt)
                lib.rtcb200Intersect1MDevice(m.sc, C.c_void_p(prim.data_ptr()), prim.shape[0], C.byref(lib.args()), C.c_void_p(stream.cuda_stream))
                torch.cuda.synchronize()
                hits = torch.empty((args.rays, 24), dtype=torch.float32, device=devt)
                for c0 in range(0, args.rays, 1 << 22):
                    ids = torch.arange(c0, min(c0 + (1 << 22), args.rays), device=devt, dtype=torch.int64)
                    hits[c0:c0 + len(ids)] = bench.bounce_rays(prim, ids)
                del prim
                lib.rtcb200Intersect1MDevice(m.sc, C.c_void_p(hits.data_ptr()), args.rays, C.byref(lib.args()), C.c_void_p(stream.cuda_stream))
                torch.cuda.synchronize()
            out = {k: torch.empty((3, args.rays), dtype=torch.float32, device=devt) for k in ("P", "dPdu", "dPdv")}

            def interp():
                lib.interpolate_hits(m.sc, hits, RTC_BUFFER_TYPE_VERTEX, 0, 3, want=("P", "dPdu", "dPdv"), stream=stream, out=out)
            i1, _, _ = timed(interp, stream)
            i2, _, _ = timed(interp, stream)
            lib.check(dev)
            if rep:
                times[name]["commit_event"].append(ce)
                times[name]["commit_wall"].append(cw)
                times[name]["interp_first"].append(i1)
                times[name]["interp_second"].append(i2)
            results[name] = torch.cat([out[k].view(torch.int32).reshape(-1) for k in ("P", "dPdu", "dPdv")]).cpu()
            m.release()
            del out
            torch.cuda.empty_cache()
    nhits = int((hits.view(torch.int32)[:, 18] != -1).sum().item())
    del hits
    torch.cuda.empty_cache()
    res = {"triangles": len(t), "rays": args.rays, "hits": nhits, "interpolated_equal": bool(torch.equal(results["host"], results["device"]))}
    for n, x in times.items():
        res[n] = {k: stat(vals) for k, vals in x.items()}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--frames", type=int, default=10)
    ap.add_argument("--phi-small", type=int, default=500, help="createTriangleSphere(P) of (a) and (b): 998 k triangles at 500")
    ap.add_argument("--phi", type=int, default=1581)
    ap.add_argument("--rays", type=int, default=64 << 20, help="rays of (d)'s headline stream")
    ap.add_argument("--frame-rays", type=int, default=1 << 20)
    args = ap.parse_args()
    lib = embree_b200.load()
    dev = lib.new_device(None)
    out = {"metric": "geometry from device buffers vs host buffers", "gpu": gpu_info(), "reps": args.reps, "frames": args.frames}
    v, t = scenes.triangle_sphere(args.phi_small)
    v = np.asarray(v, np.float32).reshape(-1, 3)
    t = np.asarray(t, np.uint32).reshape(-1, 3)
    rng = np.random.RandomState(1)
    org = rng.uniform(-2.0, 2.0, (args.frame_rays, 3))
    rh = make_rayhits(org, rng.uniform(-0.8, 0.8, (args.frame_rays, 3)) - org)
    rays = torch.from_numpy(rh.view(np.float32).reshape(-1, 24).copy()).cuda()
    out["a_refit"] = frames(lib, dev, v, t, rays, args, RTC_BUILD_QUALITY_MEDIUM, RTC_BUILD_QUALITY_REFIT, RTC_SCENE_FLAG_DYNAMIC, 2)
    out["b_rebuild_low"] = frames(lib, dev, v, t, rays, args, RTC_BUILD_QUALITY_LOW, RTC_BUILD_QUALITY_MEDIUM, RTC_SCENE_FLAG_DYNAMIC, 0)
    out["b_rebuild_medium"] = frames(lib, dev, v, t, rays, args, RTC_BUILD_QUALITY_MEDIUM, RTC_BUILD_QUALITY_MEDIUM, RTC_SCENE_FLAG_DYNAMIC, 1)
    del rays
    out["cd_first_commit_and_interp"] = first_commit_and_interp(lib, dev, args)
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))
    lib.rtcReleaseDevice(dev)


if __name__ == "__main__":
    main()
