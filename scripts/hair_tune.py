"""A/B of the leaf-test batching and grid keys of the curve / point kernels (rtcb200SetTuning) on bench.py's fur ball (flat and round
Bezier curves) and point scenes, alternating the settings in one process.  Prints Mrays/s per setting:
hair [camera closest, camera any, incoherent closest, incoherent any], points [closest, any] per kind.

    python scripts/hair_tune.py
"""
import sys
import types

import torch

sys.path.insert(0, '.')
import bench  # noqa: E402
import embree_b200  # noqa: E402

lib = embree_b200.load()
dev = lib.new_device("verbose=0")
devt = torch.device("cuda:0")
stream = torch.cuda.current_stream().cuda_stream
args = types.SimpleNamespace(no_cpu=True)
SHIPPED = dict(curve_batch_min=32, curve_wait_max=24, curve_blocks_per_sm=6, point_batch_min=24, point_wait_max=16, blocks_per_sm=8)
SETTINGS = (("shipped", SHIPPED),
            ("curves 24/16, 8 CTAs", dict(SHIPPED, curve_batch_min=24, curve_wait_max=16, curve_blocks_per_sm=8)),
            ("points 32/24", dict(SHIPPED, point_batch_min=32, point_wait_max=24)),
            ("points 16/8", dict(SHIPPED, point_batch_min=16, point_wait_max=8)),
            ("points 32/24, 6 CTAs", dict(SHIPPED, point_batch_min=32, point_wait_max=24, blocks_per_sm=6)))
for rep in range(2):
    for name, cfg in SETTINGS:
        for k, v in cfg.items():
            assert lib.rtcb200SetTuning(k.encode(), v) == 0, k
        row = {}
        for rnd in (False, True):
            o = bench.hair_leg(lib, dev, devt, stream, args, rnd=rnd)
            row["round" if rnd else "flat"] = [round(o[r][m], 1) for r in ("camera_1080p", "incoherent") for m in ("Mrays_per_s", "occluded_Mrays_per_s")]
        o = bench.point_leg(lib, dev, devt, stream, args)
        row["points"] = [round(o[k][m], 1) for k in ("sphere", "disc", "oriented_disc") for m in ("Mrays_per_s", "occluded_Mrays_per_s")]
        print(rep, name, row, flush=True)
