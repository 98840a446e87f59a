"""The quantised slab test (rt_core.cuh node_hitmask) must never cull a child box that exact arithmetic says the ray
enters.  Its rounding error is largest where every hit depends on it: a child face that lies exactly on a grid line of
the node's quantisation (dyadic coordinates: integers, powers of two, axis-aligned architecture, voxels, terrain) and a
ray origin inside a large node, far from the node's origin corner and close to that face (bounce rays start on a
surface).  These tests build such scenes -- a closed box whose faces are grids of triangles, quads or points, and a
city of integer blocks -- and require that the traversal loses no hit the oracle finds: on the CPU through the host
instantiation of the traversal (tests/emu), on the GPU through the library.  A direct property test checks
node_hitmask against an exact float64 slab test over randomised nodes and rays."""
import ctypes as C

import numpy as np
import pytest

from embree_b200.rtc import RTC_BUILD_QUALITY_LOW, RTC_BUILD_QUALITY_MEDIUM, make_rayhits, rays_of
from tests.parity import TIE_ULPS, compare_hits, explain_hit_miss, point_disagreements

MISS = 0xFFFFFFFF


# ---- scenes ------------------------------------------------------------------------------------------------------------

def grid_box(n, lo, hi, quads=False):
    """The closed box [lo, hi]^3, every face an n x n grid of quads (each split into two triangles unless `quads`).
    Returns (vertices[nv,3] f32, indices[nt,3] or [nq,4] u32); vertices are duplicated along the box's edges."""
    vs, ts = [], []
    g = np.linspace(lo, hi, n + 1).astype(np.float32)
    for axis in range(3):
        for side in (lo, hi):
            a, b = [k for k in range(3) if k != axis]
            U, V = np.meshgrid(g, g, indexing="ij")
            P = np.zeros((n + 1, n + 1, 3), np.float32)
            P[..., axis] = side
            P[..., a] = U
            P[..., b] = V
            base = sum(len(x) for x in vs)
            vs.append(P.reshape(-1, 3))
            idx = np.arange((n + 1) ** 2).reshape(n + 1, n + 1) + base
            q0, q1, q2, q3 = idx[:-1, :-1], idx[1:, :-1], idx[1:, 1:], idx[:-1, 1:]
            if quads:
                ts.append(np.stack([q0, q1, q2, q3], -1).reshape(-1, 4))
            else:
                ts.append(np.stack([q0, q1, q2], -1).reshape(-1, 3))
                ts.append(np.stack([q0, q2, q3], -1).reshape(-1, 3))
    return np.concatenate(vs), np.concatenate(ts).astype(np.uint32)


def box_grid_points(n, lo, hi):
    """The grid crossings of grid_box(n, lo, hi)'s faces as sphere points of radius a quarter grid step: (vertices4, crossings)."""
    v, _ = grid_box(n, lo, hi)
    v = np.unique(v, axis=0)
    r = np.full((len(v), 1), (hi - lo) / n / 4, np.float32)
    return np.concatenate([v, r], 1).astype(np.float32), v


def grid_city(seed, size=64, lot=8):
    """An integer-coordinate ground plane [-size, size]^2 at z = 0 (one quad per unit cell, two triangles each) and one
    axis-aligned block with integer corners and extents standing on each lot x lot square of it (10 triangles each:
    the blocks neither overlap each other nor the ground, so no two faces are coplanar)."""
    rng = np.random.RandomState(seed)
    g = np.arange(-size, size + 1, dtype=np.float32)
    X, Y = np.meshgrid(g, g, indexing="ij")
    vs = [np.stack([X, Y, np.zeros_like(X)], -1).reshape(-1, 3)]
    m = 2 * size + 1
    idx = np.arange(m * m).reshape(m, m)
    q0, q1, q2, q3 = idx[:-1, :-1], idx[1:, :-1], idx[1:, 1:], idx[:-1, 1:]
    ts = [np.stack([q0, q1, q2], -1).reshape(-1, 3), np.stack([q0, q2, q3], -1).reshape(-1, 3)]
    corners = np.array([[i & 1, (i >> 1) & 1, (i >> 2) & 1] for i in range(8)], np.float32)
    faces = np.array([[4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6],
                      [0, 2, 6], [0, 6, 4], [1, 5, 7], [1, 7, 3]], np.uint32)        # corner i = (x, y, z) bits of i; no bottom
    boxes = []
    for cx in range(-size, size, lot):
        for cy in range(-size, size, lot):
            ext = np.array([rng.randint(1, lot - 1), rng.randint(1, lot - 1), rng.randint(1, 33)], np.float32)
            lo = np.array([cx + rng.randint(1, lot - ext[0] + 1), cy + rng.randint(1, lot - ext[1] + 1), 0], np.float32)
            base = sum(len(x) for x in vs)
            vs.append(lo + corners * ext)
            ts.append(faces + base)
            boxes.append((lo, lo + ext))
    return np.concatenate(vs).astype(np.float32), np.concatenate(ts).astype(np.uint32), boxes


# ---- rays --------------------------------------------------------------------------------------------------------------

def rays_at_face_crossings(rng, n, lo, hi, count, jitter=1e-6):
    """Origins inside the box, each ray aimed at a grid crossing of a face: exactly for half the rays, jittered by
    `jitter` x the box's extent for the other half."""
    org = rng.uniform(lo + 0.01 * (hi - lo), hi - 0.01 * (hi - lo), (count, 3)).astype(np.float32)
    tgt = lo + (hi - lo) * rng.randint(0, n + 1, (count, 3)) / n
    face = rng.randint(0, 3, count)
    tgt[np.arange(count), face] = np.where(rng.rand(count) < 0.5, lo, hi)
    tgt = tgt + rng.normal(scale=jitter * (hi - lo), size=tgt.shape) * (rng.rand(count, 1) < 0.5)
    return make_rayhits(org, (tgt - org).astype(np.float32))


def axis_rays(rng, n, lo, hi, count):
    """Origins inside the box on interior grid planes, with one or two direction components exactly zero: they run
    along the grid lines of the faces they hit.  (A ray that lies in a face's own plane touches it only tangentially:
    whether the clamped direction of rcp_safe leaves or enters the box there is a matter of rounding.)"""
    org = rng.uniform(lo + 0.01 * (hi - lo), hi - 0.01 * (hi - lo), (count, 3))
    grid = lo + (hi - lo) * rng.randint(1, n, (count, 3)) / n
    d = rng.normal(size=(count, 3))
    k = rng.randint(0, 3, count)
    two = rng.rand(count) < 0.5
    for a in range(3):
        zero = (k == a) | (two & (k == (a + 1) % 3))
        d[zero, a] = 0.0
        org[zero, a] = grid[zero, a]
    return make_rayhits(org.astype(np.float32), d.astype(np.float32))


def bounce_rays(rng, first):
    """Secondary rays from the hits of `first` as pathstream's bounce kernel makes them: P = org + t dir, pushed off the
    surface by eps = 32 FLT_EPSILON max(|P|, t) along the face-forward normal, tnear = eps, a random direction in that
    hemisphere."""
    hit = first["geomID"] != MISS
    f = first[hit]
    o = np.stack([f["org_x"], f["org_y"], f["org_z"]], 1)
    d = np.stack([f["dir_x"], f["dir_y"], f["dir_z"]], 1)
    t = f["tfar"][:, None]
    P = (o + t * d).astype(np.float32)
    eps = (np.float32(32 * 1.19209e-07) * np.maximum(np.abs(P).max(1), f["tfar"])).astype(np.float32)
    ng = np.stack([f["Ng_x"], f["Ng_y"], f["Ng_z"]], 1).astype(np.float32)
    ng /= np.linalg.norm(ng, axis=1, keepdims=True)
    ng[(ng * d).sum(1) >= 0] *= -1
    wi = rng.normal(size=ng.shape).astype(np.float32)
    wi[(wi * ng).sum(1) < 0] *= -1
    r = make_rayhits((P + eps[:, None] * ng).astype(np.float32), wi)
    r["tnear"] = eps
    return r


def box_rays(seed, n, lo, hi, count, trace_first):
    """Face-crossing rays, axis-parallel rays and bounce rays from the first two sets' hits (trace_first(rays) -> hits)."""
    rng = np.random.RandomState(seed)
    a = rays_at_face_crossings(rng, n, lo, hi, count)
    b = axis_rays(rng, n, lo, hi, count // 20)
    first = np.concatenate([a, b])
    return np.concatenate([first, bounce_rays(rng, trace_first(first.copy()))[: count // 2]])


def city_rays(seed, boxes, count, trace_first):
    """Origins in the air between the blocks aimed at block corners (exactly or jittered), and bounce rays."""
    rng = np.random.RandomState(seed)
    lo = np.array([b[0] for b in boxes])
    hi = np.array([b[1] for b in boxes])
    k = rng.randint(0, len(boxes), count)
    corner = np.where(rng.rand(count, 3) < 0.5, lo[k], hi[k]).astype(np.float64)
    corner += rng.normal(scale=1e-5, size=corner.shape) * (rng.rand(count, 1) < 0.5)
    org = rng.uniform([-64, -64, 0.5], [64, 64, 40], (count, 3)).astype(np.float32)
    first = make_rayhits(org, (corner - org).astype(np.float32))
    return np.concatenate([first, bounce_rays(rng, trace_first(first.copy()))[: count // 2]])


BOXES = [(64, 0.0, 64.0), (64, -32.0, 32.0), (50, 1000.0, 1100.0), (128, 0.0, 1.0), (16, 1000.0, 1001.0),
         (32, -32.0, 992.0), (64, 1e5, 1e5 + 1024.0)]
BOX_IDS = [f"n{n}_{lo:g}_{hi:g}" for (n, lo, hi) in BOXES]


# ---- CPU: the host instantiation of the traversal --------------------------------------------------------------------

def _emu_trace(emu, v, t, rays, policy, robust, occluded=False):
    v = np.ascontiguousarray(v, np.float32)
    t = np.ascontiguousarray(t, np.uint32)
    h = emu.emu_build(v.ctypes.data, len(v), t.ctypes.data, len(t), 0, 0xFFFFFFFF, policy | (0x100 if robust else 0))
    emu.emu_trace(h, rays.ctypes.data, len(rays), 1 if occluded else 0, None)
    emu.emu_free(h)
    return rays


def nearer_hits(oracle, rays, want, got, single_prim_scene):
    """Rays on which both sides hit, at distances more than TIE_ULPS apart, on different primitives.  Each is explained
    only when this side's hit is the nearer one and the reference's arithmetic accepts that primitive alone with
    bit-equal t, u, v: the reference's box test, which does not bound its rounding error, culled it in the full scene.
    A farther hit would be a nearer one lost.  Returns (such rays, unexplained ones)."""
    both = (want["geomID"] != MISS) & (got["geomID"] != MISS)
    ulps = np.abs(want["tfar"].view(np.int32).astype(np.int64) - got["tfar"].view(np.int32).astype(np.int64))
    differ = both & (ulps > TIE_ULPS) & ((want["primID"] != got["primID"]) | (want["geomID"] != got["geomID"]) |
                                          (want["instID"] != got["instID"]))
    bad = 0
    for i in np.nonzero(differ)[0]:
        sc = single_prim_scene(int(got["geomID"][i]), int(got["primID"][i]), int(got["instID"][i]))
        r = rays[i:i + 1].copy()
        sc.trace(r)
        same = all(r[f].view(np.uint32)[0] == got[f].view(np.uint32)[i] for f in ("tfar", "u", "v"))
        bad += 0 if (got["tfar"][i] < want["tfar"][i] and r["geomID"][0] != MISS and same) else 1
        sc.free()
    return int(differ.sum()), bad


def check_against_oracle(oracle, v, t, rays, want, got, robust, closed):
    """No hit of the oracle is lost; in fast mode every extra hit is the reference's own triangle arithmetic accepting
    the primitive alone (explain_hit_miss); in robust mode inside a closed box, every miss is an oracle miss too."""
    meshes = [(v, t, 0, 0xFFFFFFFF)]
    rep = compare_hits(want, got, 1e-4, meshes=meshes)
    one = lambda g_, p_, i_: oracle.scene([(v, t[p_:p_ + 1], 0, 0xFFFFFFFF)], robust=robust)   # noqa: E731
    lost, unexplained = explain_hit_miss(oracle, rays, want, got, one)
    nearer, unexplained_nearer = nearer_hits(oracle, rays, want, got, one)
    assert lost == 0 and unexplained == 0 and unexplained_nearer == 0 and rep["id_mismatch"] == nearer, \
        (rep, lost, unexplained, nearer, unexplained_nearer)
    if robust and closed:
        escaped = (got["geomID"] == MISS) & (want["geomID"] != MISS)
        assert not escaped.any(), np.nonzero(escaped)[0][:10]
    return rep


@pytest.mark.parametrize("policy", [0, 3])
@pytest.mark.parametrize("robust", [False, True])
@pytest.mark.parametrize("box", BOXES, ids=BOX_IDS)
def test_emu_grid_box_loses_no_hit(emu, oracle, box, robust, policy):
    n, lo, hi = box
    v, t = grid_box(n, lo, hi)
    osc = oracle.scene([(v, t, 0, 0xFFFFFFFF)], robust=robust)
    rays = box_rays(7, n, lo, hi, 40000, lambda r: osc.trace(r, nthreads=8))
    want = osc.trace(rays.copy(), nthreads=8)
    got = _emu_trace(emu, v, t, rays.copy(), policy, robust)
    rep = check_against_oracle(oracle, v, t, rays, want, got, robust, closed=True)
    assert rep["hits"] > 0.6 * len(rays), rep      # the reference's own arithmetic misses some rays aimed exactly at a vertex
    occ = _emu_trace(emu, v, t, rays_of(rays), policy, robust, occluded=True)
    assert ((occ["tfar"] == -np.inf) == (got["geomID"] != MISS)).all()
    osc.free()


@pytest.mark.parametrize("policy", [0, 3])
@pytest.mark.parametrize("robust", [False, True])
def test_emu_grid_city_loses_no_hit(emu, oracle, robust, policy):
    v, t, boxes = grid_city(11)
    osc = oracle.scene([(v, t, 0, 0xFFFFFFFF)], robust=robust)
    rays = city_rays(12, boxes, 40000, lambda r: osc.trace(r, nthreads=8))
    want = osc.trace(rays.copy(), nthreads=8)
    got = _emu_trace(emu, v, t, rays.copy(), policy, robust)
    rep = check_against_oracle(oracle, v, t, rays, want, got, robust, closed=False)
    assert rep["hits"] > 0.5 * len(rays), rep
    osc.free()


# ---- CPU: node_hitmask against an exact slab test --------------------------------------------------------------------

def random_nodes_and_rays(seed, n_nodes, per_node):
    """n_nodes nodes of 1-8 child boxes and per_node rays each.  Grid steps g = 2^-18 .. 2^2 (node extents ~2^-10 .. 2^10),
    node origins up to 1e5 where float32 can hold them on that grid; children on grid lines (half the nodes) or not; ray
    origins inside the node near its origin corner, near its far corner, or outside; rays aimed exactly at a corner, an
    edge or a face of a random child; near-axis-parallel directions (components 0, +-1e-18 = rcp_safe's clamp, 1e-19,
    1e-7 x the others); tfar windows that end exactly on the aimed-at face (or one float step either side)."""
    rng = np.random.RandomState(seed)
    k = rng.randint(-18, 3, n_nodes)
    g = np.ldexp(1.0, k)
    p = rng.uniform(-1e5, 1e5, (n_nodes, 3))
    p = np.clip(np.round(p / g[:, None]), -(2 ** 22), 2 ** 22) * g[:, None]
    nch = rng.randint(1, 9, n_nodes)
    snapped = rng.rand(n_nodes) < 0.5
    i0 = rng.randint(0, 250, (n_nodes, 8, 3))
    i1 = np.minimum(i0 + rng.randint(0, 80, (n_nodes, 8, 3)), 255)
    f0 = np.where(snapped[:, None, None], i0, i0 + rng.rand(n_nodes, 8, 3))
    f1 = np.where(snapped[:, None, None], i1, np.maximum(i1 - rng.rand(n_nodes, 8, 3), f0))
    lo = (p[:, None, :] + f0 * g[:, None, None]).astype(np.float32)
    hi = (p[:, None, :] + f1 * g[:, None, None]).astype(np.float32)
    hi = np.maximum(hi, lo)
    used = np.arange(8)[None, :] < nch[:, None]
    nlo = np.where(used[..., None], lo, np.inf).min(1).astype(np.float64)
    nhi = np.where(used[..., None], hi, -np.inf).max(1).astype(np.float64)

    R = per_node
    child = (rng.rand(n_nodes, R) * nch[:, None]).astype(int)
    clo = np.take_along_axis(lo, child[..., None], 1).astype(np.float64)
    chi = np.take_along_axis(hi, child[..., None], 1).astype(np.float64)
    # target: a corner (3 axes on a face), an edge (2) or a face point (1) of the child
    on = rng.rand(n_nodes, R, 3) < rng.choice([1.0, 0.67, 0.34], (n_nodes, R))[..., None]
    side = rng.rand(n_nodes, R, 3) < 0.5
    tgt = np.where(on, np.where(side, clo, chi), clo + rng.rand(n_nodes, R, 3) * (chi - clo))
    ext = (nhi - nlo)[:, None, :]
    where = rng.randint(0, 3, (n_nodes, R))
    near_p = nlo[:, None, :] + rng.rand(n_nodes, R, 3) * 0.05 * ext
    near_far = nhi[:, None, :] - rng.rand(n_nodes, R, 3) * 0.05 * ext
    u = rng.normal(size=(n_nodes, R, 3))
    u /= np.linalg.norm(u, axis=-1, keepdims=True)
    outside = 0.5 * (nlo + nhi)[:, None, :] + u * ext.max(-1, keepdims=True) * rng.uniform(1, 20, (n_nodes, R, 1))
    org = np.select([where[..., None] == 0, where[..., None] == 1], [near_p, near_far], outside).astype(np.float32)
    d = (tgt - org) * 10.0 ** rng.uniform(-3, 3, (n_nodes, R, 1))
    # near-axis-parallel directions: one or two components replaced; the origin moves onto the aimed-at plane there
    flat = rng.rand(n_nodes, R) < 0.25
    tiny = rng.choice([0.0, 1e-18, -1e-18, 1e-19, -1e-19, 1e-7], (n_nodes, R, 3))
    tiny = np.where(tiny == 1e-7, 1e-7 * np.abs(d).max(-1, keepdims=True), tiny)
    ax = rng.rand(n_nodes, R, 3) < 0.4
    repl = flat[..., None] & ax
    d = np.where(repl, tiny, d).astype(np.float32)
    org = np.where(repl, tgt, org).astype(np.float32)
    tnear = np.where(rng.rand(n_nodes, R) < 0.1, rng.rand(n_nodes, R), 0.0).astype(np.float32)
    tfar = np.full((n_nodes, R), np.inf, np.float32)
    # tfar ends on the aimed-at face: the exact distance along one axis the target lies on, rounded, +- one step
    win = rng.rand(n_nodes, R) < 0.3
    a = np.argmax(on, -1)
    oa = np.take_along_axis(org, a[..., None], -1)[..., 0].astype(np.float64)
    da = np.take_along_axis(d, a[..., None], -1)[..., 0].astype(np.float64)
    ta = np.take_along_axis(tgt, a[..., None], -1)[..., 0]
    with np.errstate(divide="ignore", invalid="ignore"):
        tf = ((ta - oa) / np.where(np.abs(da) < 1e-18, 1e-18, da)).astype(np.float32)
    step = rng.randint(-1, 2, (n_nodes, R))
    tf = np.where(step < 0, np.nextafter(tf, np.float32(-np.inf)), np.where(step > 0, np.nextafter(tf, np.float32(np.inf)), tf))
    tfar = np.where(win & np.isfinite(tf) & (tf > 0), tf, tfar).astype(np.float32)
    boxes = np.concatenate([lo, hi], -1).astype(np.float32)
    rays = np.concatenate([org, tnear[..., None], d, tfar[..., None]], -1).astype(np.float32)
    return boxes, nch, rays


def exact_slab(boxes, nch, rays):
    """The slab test in float64 on the float32 inputs: bit c of the result is set when child c's interval
    [max(near planes, tnear), min(far planes, tfar)] is non-empty.  Direction components below 1e-18 in magnitude are
    replaced by +1e-18 first, as rcp_safe defines the ray's reciprocal direction."""
    b = boxes.astype(np.float64)[:, None, :, :]                      # node, -, child, 6
    r = rays.astype(np.float64)[:, :, None, :]                       # node, ray, -, 8
    o, d = r[..., 0:3], r[..., 4:7]
    inv = 1.0 / np.where(np.abs(d) < 1e-18, 1e-18, d)
    t0, t1 = (b[..., 0:3] - o) * inv, (b[..., 3:6] - o) * inv
    tmin = np.maximum(np.minimum(t0, t1).max(-1), np.maximum(r[..., 3], 0.0))
    tmax = np.minimum(np.maximum(t0, t1).min(-1), np.maximum(r[..., 7], 0.0))
    hit = (tmin <= tmax) & (np.arange(8)[None, None, :] < nch[:, None, None])
    return (hit * (1 << np.arange(8))[None, None, :]).sum(-1).astype(np.uint32)


def test_node_hitmask_never_culls_an_entered_child(emu):
    """Over 2^20 randomised (node, ray) cases, every child that the exact slab test says the ray enters is in
    node_hitmask's result."""
    emu.emu_node_hitmask.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_uint64, C.c_void_p]
    n_nodes, per_node = 16384, 64
    boxes, nch, rays = random_nodes_and_rays(3, n_nodes, per_node)
    want = exact_slab(boxes, nch, rays)
    got = np.zeros((n_nodes, per_node), np.uint32)
    for i in range(n_nodes):
        emu.emu_node_hitmask(boxes[i].ctypes.data, int(nch[i]), rays[i].ctypes.data, per_node, got[i].ctypes.data)
    culled = (want & ~got) != 0
    assert want.any() and (np.bitwise_count(want).sum() > 0.3 * want.size)
    assert culled.sum() == 0, (int(culled.sum()), [(int(i), int(j)) for i, j in zip(*np.nonzero(culled))][:10])


# ---- GPU: the library --------------------------------------------------------------------------------------------------

QUALITIES = [RTC_BUILD_QUALITY_LOW, RTC_BUILD_QUALITY_MEDIUM]


def _gpu_check(lib, sc, oracle, osc, rays, robust, closed, single_prim_scene):
    """Intersect through '1M' (all rays) and '16' (a slice), occluded against intersect, against the oracle."""
    want = osc.trace(rays.copy(), nthreads=16)
    got = lib.intersect(sc, rays.copy(), "1M")
    rep = compare_hits(want, got, 1e-4)          # ties: the same distance within TIE_ULPS (rays aimed at grid crossings and box edges)
    lost, unexplained = explain_hit_miss(oracle, rays, want, got, single_prim_scene)
    nearer, unexplained_nearer = nearer_hits(oracle, rays, want, got, single_prim_scene)
    assert lost == 0 and unexplained == 0 and unexplained_nearer == 0 and rep["id_mismatch"] <= nearer, \
        (rep, lost, unexplained, nearer, unexplained_nearer)
    assert rep["max_rel_t"] <= 1e-4 and rep["max_abs_uv"] <= 1e-4, rep
    if robust and closed:
        assert not ((got["geomID"] == MISS) & (want["geomID"] != MISS)).any(), rep
    sub = rays[:4096]
    got16 = lib.intersect(sc, sub.copy(), "16")
    assert (got16.view(np.uint8) == got[:4096].view(np.uint8)).all()
    occ = lib.occluded(sc, rays_of(rays), "1M")
    assert ((occ["tfar"] == -np.inf) == (got["geomID"] != MISS)).all()
    return rep


@pytest.mark.gpu
@pytest.mark.parametrize("robust", [False, True])
@pytest.mark.parametrize("quality", QUALITIES)
@pytest.mark.parametrize("box", BOXES + ["city"], ids=BOX_IDS + ["city"])
def test_gpu_grid_scenes_lose_no_hit(b200, oracle, box, quality, robust):
    from tests.test_gpu_parity import build_scene
    lib, dev = b200
    if box == "city":
        v, t, boxes = grid_city(11)
    else:
        n, lo, hi = box
        v, t = grid_box(n, lo, hi)
    meshes = [(v, t, 0, 0xFFFFFFFF)]
    sc, keep = build_scene(lib, dev, meshes, quality, flags=4 if robust else 0)
    osc = oracle.scene(meshes, robust=robust)
    first = lambda r: osc.trace(r, nthreads=16)   # noqa: E731
    rays = city_rays(12, boxes, 100000, first) if box == "city" else box_rays(7, n, lo, hi, 100000, first)
    _gpu_check(lib, sc, oracle, osc, rays, robust, box != "city",
               lambda g_, p_, i_: oracle.scene([(v, t[p_:p_ + 1], 0, 0xFFFFFFFF)], robust=robust))
    osc.free()
    lib.rtcReleaseScene(sc)


@pytest.mark.gpu
@pytest.mark.parametrize("robust", [False, True])
def test_gpu_large_grid_box(b200, oracle, robust):
    """256 x 256 quads per face (786 k triangles): both phases of the SAH builder and deep trees."""
    from tests.test_gpu_parity import build_scene
    lib, dev = b200
    n, lo, hi = 256, -128.0, 128.0
    v, t = grid_box(n, lo, hi)
    meshes = [(v, t, 0, 0xFFFFFFFF)]
    sc, keep = build_scene(lib, dev, meshes, RTC_BUILD_QUALITY_MEDIUM, flags=4 if robust else 0)
    osc = oracle.scene(meshes, robust=robust)
    rays = box_rays(8, n, lo, hi, 200000, lambda r: osc.trace(r, nthreads=16))
    _gpu_check(lib, sc, oracle, osc, rays, robust, True,
               lambda g_, p_, i_: oracle.scene([(v, t[p_:p_ + 1], 0, 0xFFFFFFFF)], robust=robust))
    osc.free()
    lib.rtcReleaseScene(sc)


@pytest.mark.gpu
@pytest.mark.parametrize("robust", [False, True])
def test_gpu_grid_box_instanced_and_quads(b200, oracle, robust):
    """The box as the child scene of an instance that scales by 2 and translates by 1000: the transform is dyadic, so
    the rays taken into object space keep their grid alignment.  With RTC_SCENE_FLAG_ROBUST, the box as QUAD geometry
    as well.  (In fast mode some extra hits of rays aimed exactly at a quad's corner are not reproduced bit-exactly by
    the oracle's scene of that quad alone, as explain_hit_miss requires; that is not explained yet.)"""
    from tests.test_gpu_parity import build_scene
    lib, dev = b200
    n, lo, hi = 64, -32.0, 32.0
    vt, t = grid_box(n, lo, hi)
    child, keep2 = build_scene(lib, dev, [(vt, t, 0, 0xFFFFFFFF)], RTC_BUILD_QUALITY_MEDIUM, flags=4 if robust else 0)
    xfm = np.array([2, 0, 0, 0, 2, 0, 0, 0, 2, 1000, 1000, 1000], np.float32)
    top = lib.rtcNewScene(dev)
    if robust:
        lib.rtcSetSceneFlags(top, 4)
    lib.add_instance(dev, top, child, xfm, mask=0xFFFFFFFF, geom_id=0)
    lib.rtcCommitScene(top)
    lib.check(dev)
    oc = oracle.scene([(vt, t, 0, 0xFFFFFFFF)], robust=robust)
    ot = oracle.scene([], robust=robust, instances=[(oc, xfm, 0, 0xFFFFFFFF)])
    wlo, whi = 1000 + 2 * lo, 1000 + 2 * hi
    rays = box_rays(10, n, wlo, whi, 100000, lambda r: ot.trace(r, nthreads=16))

    def one_tri_instanced(g_, p_, i_):
        c = oracle.scene([(vt, t[p_:p_ + 1], 0, 0xFFFFFFFF)], robust=robust)
        return oracle.scene([], robust=robust, instances=[(c, xfm, 0, 0xFFFFFFFF)])
    _gpu_check(lib, top, oracle, ot, rays, robust, True, one_tri_instanced)
    ot.free()
    oc.free()
    lib.rtcReleaseScene(top)
    lib.rtcReleaseScene(child)
    if not robust:
        return
    v, q = grid_box(n, lo, hi, quads=True)
    meshes = [(v, q, 0, 0xFFFFFFFF)]
    sc, keep = build_scene(lib, dev, meshes, RTC_BUILD_QUALITY_MEDIUM, flags=4 if robust else 0)
    osc = oracle.scene(meshes, robust=robust)
    rays = box_rays(9, n, lo, hi, 100000, lambda r: osc.trace(r, nthreads=16))
    _gpu_check(lib, sc, oracle, osc, rays, robust, True,
               lambda g_, p_, i_: oracle.scene([(v, q[p_:p_ + 1], 0, 0xFFFFFFFF)], robust=robust))
    osc.free()
    lib.rtcReleaseScene(sc)


@pytest.mark.gpu
def test_gpu_grid_points(b200, oracle):
    """Sphere points on the grid crossings of the box's faces (their boxes' faces lie on the grid too), rays from inside
    aimed at the points' extreme points along the axes: the point kernels run the same node test."""
    lib, dev = b200
    n, lo, hi = 32, 992.0, 1024.0
    pv, c = box_grid_points(n, lo, hi)
    sc = lib.rtcNewScene(dev)
    keep = lib.add_points(dev, sc, pv, "sphere", mask=0xFFFFFFFF, geom_id=0)
    lib.rtcCommitScene(sc)
    lib.check(dev)
    osc = oracle.scene([], points=[(pv, "sphere", None, 0, 0xFFFFFFFF)])
    rng = np.random.RandomState(13)
    m = 100000
    org = rng.uniform(lo + 1, hi - 1, (m, 3)).astype(np.float32)
    k = rng.randint(0, len(pv), m)
    tgt = c[k].astype(np.float64)
    a = rng.randint(0, 3, m)
    tgt[np.arange(m), a] += np.where(rng.rand(m) < 0.5, -1, 1) * pv[k, 3]
    rays = make_rayhits(org, (tgt - org).astype(np.float32))
    want = osc.trace(rays.copy(), nthreads=16)
    got = lib.intersect(sc, rays.copy(), "1M")
    n_differ, unexplained = point_disagreements(rays, want, got, {0: (pv, "sphere", None)})
    lost = ((want["geomID"] != MISS) & (got["geomID"] == MISS)).sum()
    assert unexplained == 0 and lost <= n_differ, (n_differ, unexplained, lost)
    assert (want["geomID"] != MISS).mean() > 0.9
    got16 = lib.intersect(sc, rays[:4096].copy(), "16")
    assert (got16.view(np.uint8) == got[:4096].view(np.uint8)).all()
    occ = lib.occluded(sc, rays_of(rays), "1M")
    assert ((occ["tfar"] == -np.inf) == (got["geomID"] != MISS)).all()
    osc.free()
    lib.rtcReleaseScene(sc)
