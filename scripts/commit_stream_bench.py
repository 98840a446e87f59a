"""Commits on a CUDA stream (rtcb200CommitSceneWithStream) against rtcCommitScene, on DESIGN section 9 (a)'s frame: a DYNAMIC REFIT
triangle mesh whose vertices (device views) a torch kernel moves, a commit, then rays traced through rtcb200Intersect1MDevice.  Two
sizes: 1 M triangles with 1 Mi rays, and 64 k triangles with 256 Ki rays, where the fixed costs of a frame weigh most.

  sync     move, torch.cuda.synchronize(), rtcCommitScene, trace                (two host round trips per frame)
  stream   move, commit on the stream, trace; one synchronise every 10 frames    (the refit returns without waiting)

Both arms run on one torch stream; they alternate, one warm-up each, then --reps repetitions of --frames frames.  Reported per
frame: wall clock (a synchronise ends each repetition) and CUDA-event time between the first and the last frame's work on the stream,
median [min, max] over the repetitions; the card's name, power limit and max SM clock read in the same run; and whether the two arms'
traced records are byte-identical frame for frame.  Prints one JSON line; writes nothing.

    python scripts/commit_stream_bench.py [--reps R] [--frames F]
"""
import argparse
import ctypes as C
import json
import math
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import embree_b200  # noqa: E402
from embree_b200 import scenes  # noqa: E402
from embree_b200.rtc import (RTC_BUFFER_TYPE_INDEX, RTC_BUFFER_TYPE_VERTEX, RTC_BUILD_QUALITY_MEDIUM, RTC_BUILD_QUALITY_REFIT,  # noqa: E402
                             RTC_FORMAT_FLOAT3, RTC_FORMAT_UINT3, RTC_GEOMETRY_TYPE_TRIANGLE, RTC_SCENE_FLAG_DYNAMIC, make_rayhits)
from scripts.device_traversal_bench import gpu_info  # noqa: E402

SYNC_EVERY = 10


def stat(x):
    return {"ms_median": float(np.median(x)), "ms_range": [float(min(x)), float(max(x))]}


class Mesh:
    """A DYNAMIC scene of one REFIT triangle mesh from device views; move(f) sets the vertices of frame f (a torch kernel)."""

    def __init__(self, lib, dev, v, t):
        self.lib = lib
        self.base = torch.from_numpy(np.ascontiguousarray(v, np.float32)).cuda()
        self.v = self.base.clone()
        self.idx = torch.from_numpy(np.ascontiguousarray(t, np.uint32).view(np.int32)).cuda()
        self.sc = lib.rtcNewScene(dev)
        lib.rtcSetSceneFlags(self.sc, RTC_SCENE_FLAG_DYNAMIC)
        lib.rtcSetSceneBuildQuality(self.sc, RTC_BUILD_QUALITY_MEDIUM)
        self.g = lib.rtcNewGeometry(dev, RTC_GEOMETRY_TYPE_TRIANGLE)
        torch.cuda.synchronize()
        lib.set_device_buffer(self.g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, self.v)
        lib.set_device_buffer(self.g, RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT3, self.idx)
        lib.rtcSetGeometryBuildQuality(self.g, RTC_BUILD_QUALITY_REFIT)
        lib.rtcCommitGeometry(self.g)
        lib.rtcAttachGeometry(self.sc, self.g)
        lib.rtcReleaseGeometry(self.g)
        lib.rtcCommitScene(self.sc)
        lib.check(dev)

    def move(self, f):
        torch.mul(self.base, 1.0 + 0.05 * math.sin(0.37 * f), out=self.v)
        self.lib.rtcUpdateGeometryBuffer(self.g, RTC_BUFFER_TYPE_VERTEX, 0)
        self.lib.rtcCommitGeometry(self.g)

    def release(self):
        self.lib.release_device_buffers(self.g)
        self.lib.rtcReleaseScene(self.sc)


def run(lib, dev, num_phi, nrays, args):
    v, t = scenes.triangle_sphere(num_phi, (0.0, 0.0, 0.0), 1.5)
    rng = np.random.RandomState(1)
    org = rng.uniform(-2.0, 2.0, (nrays, 3))
    rays = torch.from_numpy(make_rayhits(org, rng.uniform(-0.8, 0.8, (nrays, 3)) - org).view(np.uint8).copy()).cuda()
    S = torch.cuda.Stream()
    meshes = {arm: Mesh(lib, dev, v, t) for arm in ("sync", "stream")}
    outs = {arm: [torch.empty_like(rays) for _ in range(args.frames)] for arm in meshes}
    a = lib.args()
    wall = {arm: [] for arm in meshes}
    gpu = {arm: [] for arm in meshes}
    same = True
    for rep in range(args.reps + 1):
        order = ("sync", "stream") if rep % 2 == 0 else ("stream", "sync")
        for arm in order:
            m = meshes[arm]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            with torch.cuda.stream(S):
                e0.record(S)
                for f in range(args.frames):
                    m.move(f)
                    if arm == "sync":
                        torch.cuda.synchronize()
                        lib.rtcCommitScene(m.sc)
                    else:
                        lib.commit_on_stream(m.sc, S)
                    outs[arm][f].copy_(rays)
                    lib.rtcb200Intersect1MDevice(m.sc, C.c_void_p(outs[arm][f].data_ptr()), nrays, C.byref(a), C.c_void_p(S.cuda_stream))
                    if arm == "stream" and (f + 1) % SYNC_EVERY == 0:
                        S.synchronize()
                e1.record(S)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            lib.check(dev)
            if rep > 0:
                wall[arm].append((t1 - t0) * 1e3 / args.frames)
                gpu[arm].append(e0.elapsed_time(e1) / args.frames)
        same = same and all(torch.equal(x, y) for x, y in zip(outs["sync"], outs["stream"]))
    hits = int((outs["stream"][-1].view(torch.int32).view(-1, 24)[:, 18] != -1).sum())
    builder = lib.scene_stats(meshes["stream"].sc).builder
    for m in meshes.values():
        m.release()
    res = {"triangles": len(t), "rays": nrays, "hits": hits, "builder": builder, "records_equal": bool(same)}
    for arm in meshes:
        res[arm] = {"wall_per_frame": stat(wall[arm]), "gpu_per_frame": stat(gpu[arm])}
    res["wall_speedup"] = res["sync"]["wall_per_frame"]["ms_median"] / res["stream"]["wall_per_frame"]["ms_median"]
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--frames", type=int, default=50)
    args = ap.parse_args()
    assert args.frames % SYNC_EVERY == 0
    lib = embree_b200.load()
    dev = lib.new_device(None)
    out = {"gpu": gpu_info(), "frames": args.frames, "reps": args.reps,
           "1M_tris_1Mi_rays": run(lib, dev, 500, 1 << 20, args),
           "64k_tris_256Ki_rays": run(lib, dev, 128, 1 << 18, args)}
    lib.rtcReleaseDevice(dev)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
