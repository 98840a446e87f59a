"""Curve primitives at the corners of their intersectors' domain on the GPU (tests/curve_cases.py curve_edge_cases): each of the ten
curve kinds alone, at LOW and MEDIUM build quality, through every ray entry point, against the C oracle -- which is pinned to the
reference on the same rays (tests/test_oracle.py test_oracle_curve_edge_cases_vs_live_reference) and whose arithmetic the device code
repeats operation for operation (tests/test_emu_core.py test_curve_edge_cases_equal_oracle)."""
import numpy as np
import pytest

from embree_b200.rtc import RTC_BUILD_QUALITY_LOW, RTC_BUILD_QUALITY_MEDIUM, rays_of
from tests.curve_cases import CURVE_KINDS, RAY_MODES, add_curve_sets, curve_edge_cases, curve_edge_disagreements, oracle_scene
from tests.curve_exact import f64_departures

pytestmark = pytest.mark.gpu
MODES = ["1", "4", "8", "16", "1M", "4M", "8M", "16M", "1MDevice"]


def _trace(lib, sc, rays, mode, occluded=False):
    """rays through one entry point; '1MDevice': rtcb200Intersect1MDevice / rtcb200Occluded1MDevice on records in GPU memory."""
    if mode != "1MDevice":
        return lib.occluded(sc, rays, mode) if occluded else lib.intersect(sc, rays, mode)
    import ctypes as C
    import torch
    st = torch.cuda.current_stream()
    d = torch.from_numpy(rays.view(np.uint8).copy()).cuda()
    fn = lib.rtcb200Occluded1MDevice if occluded else lib.rtcb200Intersect1MDevice
    fn(sc, C.c_void_p(d.data_ptr()), len(rays), C.byref(lib.args()), C.c_void_p(st.cuda_stream))
    torch.cuda.synchronize()
    rays.view(np.uint8)[:] = d.cpu().numpy()
    return rays


def _bvh_geoms(S):
    """The curve sets as tests/bvh_check.py Geoms."""
    from tests import bvh_check as bc
    geoms = [bc.Geom(bc.FLAT_LINEAR if flat else bc.ROUND_LINEAR, gid, cv, ci, mask=mask, flags=cf) for (cv, ci, cf, gid, mask, flat) in S["curves"]]
    geoms += [bc.Geom(bc.ROUND_CUBIC if rnd else bc.FLAT_CUBIC, gid, cv, ci, mask=mask, basis={"bezier": 0, "bspline": 1, "catmull_rom": 2, "hermite": 0}[b],
                      tess=tess, tangents=tg) for (cv, ci, gid, mask, b, tess, tg, rnd) in S["cubics"]]
    return geoms


def _alone(oracle, S, gid, prim, ray):
    """The oracle's record for `ray` against curve `prim` of cubic geometry `gid` alone."""
    cv, ci, _g, mask, basis, tess, tg, rnd = [c for c in S["cubics"] if c[2] == gid][0]
    sc = oracle.scene([], cubics=[(cv, ci[prim:prim + 1], gid, mask, basis, 4 if tess is None else tess, tg, rnd)])
    out = sc.trace(ray.copy())
    sc.free()
    return out


def _folds_back(S, a, b):
    """Per ray: do the two records name points of one cubic curve's centreline that lie within the curve's largest radius of each other?
    A curve that folds back on itself (a Hermite curve from a point to the same point) meets the ray at one distance at two u, and
    which of them a traversal reports depends on the order in which the BVH offers the curve's segments."""
    from tests.curve_cases import _prim_cp, cubic_eval, kind_parts
    out = np.zeros(len(a), bool)
    if not S["cubics"]:
        return out
    basis = kind_parts("x_" + S["cubics"][0][4])[1]
    for i in np.nonzero((a["geomID"] != 0xFFFFFFFF) & (a["geomID"] == b["geomID"]) & (a["primID"] == b["primID"]))[0]:
        cp = _prim_cp(S, int(a["geomID"][i]), int(a["primID"][i]))
        P = cubic_eval(np.repeat(cp, 2, 0), basis, np.array([a["u"][i], b["u"][i]], np.float64))
        out[i] = np.linalg.norm(P[0, :3] - P[1, :3]) <= np.abs(cp[0, :, 3]).max()
    return out


@pytest.mark.parametrize("quality", [RTC_BUILD_QUALITY_LOW, RTC_BUILD_QUALITY_MEDIUM])
@pytest.mark.parametrize("kind", CURVE_KINDS)
def test_curve_edge_cases_vs_oracle(b200, oracle, kind, quality):
    """Every entry point, rtcb200Intersect1MDevice / Occluded1MDevice included, and the device-built BVH checked by tests/bvh_check.py.
    Rays across invalid primitives hit nothing; against the float64 statements of tests/curve_exact.py the device departs only where
    the oracle does (which departs only where the reference does); occluded differs from the oracle only on rays intersect differs on.
    Linear kinds and flat cubics: every record the oracle names bit-identical in t / u / v / Ng; another primitive only at a
    bit-identical t (a joint) or, on at most 1 % of the rays, where the oracle and the device traverse different leaf boxes around a round linear cone hit beyond
    its segment's solid (curve_cases.py curve_edge_disagreements).  Round cubics: the BVH holds a curve's 7 sub-segments as separate
    records, so candidates shorten tfar in another order than the oracle's whole-curve loop and the Newton start of an exit point moves
    with it: every difference must sit on a boundary rule or be that order (the device's nearer hit is what the oracle finds on that
    curve alone), and nearly all shared records stay bit-identical.  A curve that folds back on itself is met at one distance at two
    u: either may be reported.  Occluded agrees."""
    lib, dev = b200
    S = curve_edge_cases(kind)
    rays = S["rays"]
    o = oracle_scene(oracle, S)
    want = o.trace(rays.copy())
    wocc = o.trace(rays_of(rays), occluded=True)
    o.free()
    sc = lib.rtcNewScene(dev)
    lib.rtcSetSceneBuildQuality(sc, quality)
    keep = add_curve_sets(lib, dev, sc, S)
    lib.rtcCommitScene(sc)
    lib.check(dev)
    # every valid primitive of the thin, fat, far-away and tiny sets in a leaf, in a box that covers it in float64; no invalid one
    from tests.bvh_check import check_bvh
    check_bvh(lib.scene_arrays(sc), _bvh_geoms(S))
    cubic_round = kind.startswith("round_") and kind != "round_linear"
    inv = S["mode"] == RAY_MODES.index("invalid")
    _c, orc_dep = f64_departures(kind, S, rays, want)
    for mode in MODES:
        got = _trace(lib, sc, rays.copy(), mode)
        dis = curve_edge_disagreements(kind, S, rays, want, got, t_tol=1e-3 if cubic_round else 1e-4, tie_ulps=4 if cubic_round else 0)
        order = 0
        if cubic_round:        # the nearer record must be what the oracle finds on that curve alone: then only the order differs
            for i in list(dis["rows"]):
                if got["geomID"][i] != 0xFFFFFFFF and (want["geomID"][i] == 0xFFFFFFFF or got["tfar"][i] < want["tfar"][i]):
                    one = _alone(oracle, S, int(got["geomID"][i]), int(got["primID"][i]), rays[i:i + 1])
                    if one["geomID"][0] != 0xFFFFFFFF and abs(float(one["tfar"][0]) - float(got["tfar"][i])) <= 1e-3 * float(got["tfar"][i]):
                        dis["rows"].remove(i)
                        order += 1
            dis["unexplained"] -= order
        same = (got["geomID"] == want["geomID"]) & (got["primID"] == want["primID"]) & (want["geomID"] != 0xFFFFFFFF)
        exact = same.copy()
        for f in ("tfar", "u", "v", "Ng_x", "Ng_y", "Ng_z"):
            exact &= got[f].view(np.uint32) == want[f].view(np.uint32)
        self_tie = same & ~exact & (got["tfar"].view(np.uint32) == want["tfar"].view(np.uint32)) & _folds_back(S, want, got)
        print(kind, quality, mode, dict(rays=len(rays), hits=int(same.sum()), bit_exact=int(exact.sum()), self_tie=int(self_tie.sum()), order=order,
                                        **{k: v for k, v in dis.items() if k != "rows"}))
        assert dis["unexplained"] == 0, (mode, dis, [rays[i] for i in dis["rows"][:2]])
        if cubic_round:
            # seen: 98 % bit-exact, 99.6 % with the fold-back ties (Hermite curves from a point to the same point)
            assert dis["differ"] <= 0.01 * len(rays) and (exact | self_tie).sum() >= 0.99 * same.sum(), (mode, dis, int(exact.sum()), int(same.sum()))
        else:
            assert dis["differ"] == dis["beyond_the_solid"] <= 0.01 * len(rays) and (exact | self_tie).sum() == same.sum(), \
                (mode, dis, int(exact.sum()), int(same.sum()))
        assert (got["geomID"][inv] == 0xFFFFFFFF).all(), mode
        # the float64 statement: the device departs from it only where the oracle does, or on a ray the two differ on by a rule
        _c, dep = f64_departures(kind, S, rays, got)
        assert set(np.nonzero(dep & ~orc_dep)[0].tolist()) <= set(dis["differ_rows"].tolist()), mode
        occ = _trace(lib, sc, rays_of(rays), mode, occluded=True)
        assert set(np.nonzero((occ["tfar"] == -np.inf) != (wocc["tfar"] == -np.inf))[0].tolist()) <= set(dis["differ_rows"].tolist()), mode
    lib.rtcReleaseScene(sc)
    del keep
