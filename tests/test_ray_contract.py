"""The ray/triangle contract (DESIGN §3) on the product's own walk: closest hit = smallest t, ties to the smallest global triangle id, any-hit =
existence, so the answer must not depend on the tree.  `World.trace_rays` runs the frame's walk (`kjb::trace`) or a brute force over every
triangle record (the same `intersect_leaf`) on hostile rays: aimed at shared edges and vertices from near and very far, exact ties between
copies in different leaves, rays lying in node planes, hit-clipping tmin / tmax windows, NaN / Inf / zero directions, grazing rays.

  a. walk == brute force, bit for bit, on the emulator (rays beyond the conditioning limit of the culling slack, kjb_trace.cuh: a weaker check);
  b. the product's brute force == the oracle's brute force, bit for bit (an independent restatement of the triangle test);
  c. a float64 Moeller-Trumbore on the same world triangles, where float32 rounding cannot flip the answer;
  e. on the GPU: (a) on the full atrium and ruins, and the H100 == the emulator on the CPU scenes.
The oracle's own walker gets the same rays in tests/test_oracle_bvh.py."""
import ctypes as C
import functools
import numpy as np
import pytest
import conftest
import parity
from kajiya_b200 import scenes

U = 2.0 ** -24
# the conditioning limit DESIGN §3 promises: the culling slack s = k * 2^-24 of both walkers (KJB_SLAB_SLACK_K in kjb_trace.cuh,
# SLAB_SLACK in oracle/kj_scene.h) covers Moeller-Trumbore's t error up to this k.  Fixed here, so a walker with less slack fails.
SLACK_K = 16384.0
MISS = 0xffffffff
MODES = [dict(any_hit=a, cull_back=c) for a in (False, True) for c in (False, True)]
IDENTITY = np.eye(3, 4, dtype=np.float32)


# ------------------------------------------------------------------------------------------------ scenes
def _mesh(tris, mat=0):
    p = np.asarray(tris, np.float32).reshape(-1, 3)
    return dict(positions=p, normals=np.tile(np.array([[0, 1, 0]], np.float32), (len(p), 1)), indices=np.arange(len(p), dtype=np.uint32),
                material_ids=np.full(len(p), mat, np.uint32), materials=[dict(base_color=[0.6, 0.6, 0.6, 1.0], roughness=0.7)])


def tie_clusters(seed=7, n=24):
    """clusters of 8 triangles with one box centre: 5 copies of a triangle T lying in an axis plane, then 3 of a triangle W whose box is T's
    widened along the normal.  Coincident centroids make the builder halve each cluster by global id, so T's lowest copies sit in a leaf with
    a flat box and a higher copy shares a leaf with W: that leaf is entered first from either side, and its T returns the same t."""
    rs = np.random.RandomState(seed)
    tris = []
    for k in range(n):
        axis = k % 3
        c = rs.uniform(-4, 4, 3).astype(np.float32)
        a, b = [(axis + 1) % 3, (axis + 2) % 3]
        sa, sb = rs.uniform(0.3, 1.0, 2)
        lo, hi = c.copy(), c.copy()
        lo[a] -= sa; hi[a] += sa; lo[b] -= sb; hi[b] += sb
        t0, t1, t2 = lo.copy(), lo.copy(), lo.copy()
        t1[a] = hi[a]; t2[b] = hi[b]; t2[a] = hi[a]          # T: corners (lo_a, lo_b), (hi_a, lo_b), (hi_a, hi_b) in the plane axis = c
        h = rs.uniform(0.5, 2.0)
        w0, w1, w2 = t0.copy(), t1.copy(), t0.copy()
        w0[axis] -= h; w1[axis] += h; w2[b] = hi[b]; w2[axis] += h   # W: box = T's box widened by h on both sides of its plane
        tris += [np.stack([t0, t1, t2])] * 5 + [np.stack([w0, w1, w2])] * 3
    return _mesh(np.stack(tris))


def dyadic_grid(n=8, step=0.25):
    """a flat grid at y = 0 whose coordinates and every Moeller-Trumbore intermediate of the axis-aligned rays below are exact in float32"""
    tris = []
    for i in range(n):
        for j in range(n):
            x0, z0 = -1 + i * step, -1 + j * step
            a, b, c, d = (x0, 0, z0), (x0 + step, 0, z0), (x0 + step, 0, z0 + step), (x0, 0, z0 + step)
            tris += [(a, b, c), (a, c, d)] if (i + j) % 2 else [(a, b, d), (b, c, d)]
    return _mesh(np.array(tris, np.float32))


def _tr(s=1.0, t=(0.0, 0.0, 0.0)):
    return np.array([[2 * s, 0, 0, t[0]], [0, 2 * s, 0, t[1] - s], [0, 0, 2 * s, t[2]]], np.float32)   # Cornell's own transform, scaled, moved


def scene(name):
    cornell, _ = scenes.cornell_box()
    mesh = cornell[0][0]
    if name == "cornell":
        return cornell
    if name == "ruins":
        return scenes.ruins(grid=24)[0]
    if name == "atrium_20k":
        return scenes.atrium(target_tris=20000)[0]
    if name == "cornell_far":     # three instances: moved by 10^3, by 3 * 10^4, and scaled by 100
        return [(mesh, [_tr(1.0, (1e3, 1e3, -1e3)), _tr(1.0, (3e4, 0.0, 3e4)), _tr(100.0, (0.0, -300.0, 0.0))])]
    if name == "coincident":      # six coincident instances: the builder's halving fallback
        return [(mesh, [cornell[0][1][0]] * 6)]
    if name == "ties":
        return [(tie_clusters(), [IDENTITY])]
    if name == "dyadic":
        return [(dyadic_grid(), [IDENTITY])]
    raise KeyError(name)


def _start_transforms(sc):
    """other transforms with the same meshes: the world is built there, then moved to `sc`, which the refit serves"""
    return [(m, [np.asarray(t, np.float32) + np.array([[0, 0, 0, 0.75], [0, 0, 0, -0.5], [0, 0, 0, 0.25]], np.float32) for t in ts]) for m, ts in sc]


def make_world(lib, name, refit=False):
    sc = scene(name)
    _, view = scenes.cornell_box()
    w = parity.make_world(lib, _start_transforms(sc) if refit else sc, 16, 8)
    w.render_frame(**view)
    if refit:
        h = 0
        for _, ts in sc:
            for t in ts:
                w.set_instance_transform(h, t); h += 1
        w.render_frame(**view)
    return w


# ------------------------------------------------------------------------------------------------ the float64 restatement
def tri_arrays(wt):
    """v0, e1, e2 as the library stores them (e = float32(b - a)), as float64"""
    v = wt.reshape(-1, 3, 3)
    return v[:, 0].astype(np.float64), (v[:, 1] - v[:, 0]).astype(np.float64), (v[:, 2] - v[:, 0]).astype(np.float64)


def mt64(rays, v0, e1, e2, idx=None):
    """float64 Moeller-Trumbore of rays[k] against triangles idx[k] (or all): det, u, v, t, and the quantities that bound float32's error"""
    o, d = rays[:, None, 0:3].astype(np.float64), rays[:, None, 4:7].astype(np.float64)
    if idx is not None:
        v0, e1, e2 = v0[idx][:, None], e1[idx][:, None], e2[idx][:, None]
    with np.errstate(all="ignore"):
        p = np.cross(d, e2)
        det = (e1 * p).sum(-1)
        tv = o - v0
        u = (tv * p).sum(-1) / det
        q = np.cross(tv, e1)
        v = (d * q).sum(-1) / det
        t = (e2 * q).sum(-1) / det
        n = np.cross(e1, e2)
        a2 = np.linalg.norm(n, axis=-1)
        cos = np.abs(det) / (np.linalg.norm(d, axis=-1) * a2)
        shape = np.linalg.norm(e1, axis=-1) * np.linalg.norm(e2, axis=-1) / a2
        rho = np.linalg.norm(tv, axis=-1) / (np.abs(t) * np.linalg.norm(d, axis=-1))
        lmax = np.maximum(np.maximum(np.linalg.norm(e1, axis=-1), np.linalg.norm(e2, axis=-1)), np.linalg.norm(e2 - e1, axis=-1))
        bary_err = 64 * U * np.linalg.norm(tv, axis=-1) * lmax / (a2 * cos)
    return dict(det=det, u=u, v=v, t=t, cos=cos, shape=shape, rho=rho, bary_err=bary_err)


def t_error_bound(m):
    """the first-order relative error bound of float32 Moeller-Trumbore's t (kjb_trace.cuh), in units of 2^-24"""
    return 1.155 * (6 * m["rho"] + 5) * m["shape"] / m["cos"] + 2


def conditioned(rays, res, wt):
    """rays whose hit (res: trace_rays words) lies within the culling slack's limit: the walk can never cull that triangle"""
    hit = res[:, 3] != MISS
    ok = np.ones(len(rays), bool)
    if hit.any():
        v0, e1, e2 = tri_arrays(wt)
        m = mt64(rays[hit], v0, e1, e2, res[hit, 3].astype(np.int64))
        b = t_error_bound({k: x[:, 0] for k, x in m.items()})
        ok[hit] = np.nan_to_num(b, nan=np.inf) <= 0.9 * SLACK_K - 6
    return ok


# ------------------------------------------------------------------------------------------------ ray sets (generated from seeds)
def _unit(rs, n):
    d = rs.randn(n, 3)
    return d / np.linalg.norm(d, axis=1, keepdims=True)


def _rays(o, d, tmin=0.0, tmax=np.inf):
    r = np.zeros((len(o), 8), np.float32)
    r[:, 0:3] = o; r[:, 3] = tmin; r[:, 4:7] = d; r[:, 7] = tmax
    return r


def edge_rays(wt, rs, per=64, dists=(1.0, 10.0, 1e2, 1e3, 1e4)):
    """aimed at points of triangle edges (s = 0: vertices, 1/2, random) from 1 to 10^4 scene sizes away"""
    v = wt.reshape(-1, 3, 3).astype(np.float64)
    size = float(np.linalg.norm(v.reshape(-1, 3).max(0) - v.reshape(-1, 3).min(0)))
    out = []
    for dist in dists:
        for s_kind in range(3):
            k = rs.randint(0, len(v), per); e = rs.randint(0, 3, per)
            a, b = v[k, e], v[k, (e + 1) % 3]
            s = np.zeros(per) if s_kind == 0 else (np.full(per, 0.5) if s_kind == 1 else rs.rand(per))
            p = a + s[:, None] * (b - a)
            o = (p + dist * size * _unit(rs, per)).astype(np.float32)
            d = (p - o.astype(np.float64)); d /= np.linalg.norm(d, axis=1, keepdims=True)
            out.append(_rays(o, d.astype(np.float32)))
    return np.concatenate(out)


def interior_rays(wt, rs, n, dists=(1.0, 10.0, 1e2, 1e3)):
    """aimed at random interior points of random triangles"""
    v = wt.reshape(-1, 3, 3).astype(np.float64)
    size = float(np.linalg.norm(v.reshape(-1, 3).max(0) - v.reshape(-1, 3).min(0)))
    k = rs.randint(0, len(v), n)
    b = rs.dirichlet((2, 2, 2), n)
    p = (b[:, :, None] * v[k]).sum(1)
    o = (p + np.asarray(dists)[rs.randint(0, len(dists), n)][:, None] * size * _unit(rs, n)).astype(np.float32)
    d = p - o.astype(np.float64); d /= np.linalg.norm(d, axis=1, keepdims=True)
    return _rays(o, d.astype(np.float32))


def plane_rays(tree, rs, n):
    """axis-aligned rays with signed-zero components, starting exactly on a node's box plane: along the plane and across it"""
    nodes = tree["nodes"]
    if not len(nodes):
        return np.zeros((0, 8), np.float32)
    box = nodes[:, :12].view(np.float32)
    i = rs.randint(0, len(nodes), n); k = rs.randint(0, 2, n)
    lo = np.stack([box[i, 4 * k], box[i, 4 * k + 2], box[i, 8 + 2 * k]], 1)
    hi = np.stack([box[i, 4 * k + 1], box[i, 4 * k + 3], box[i, 8 + 2 * k + 1]], 1)
    o = (lo + rs.rand(n, 3).astype(np.float32) * (hi - lo)).astype(np.float32)
    a = rs.randint(0, 3, n)
    side = rs.randint(0, 2, n)
    o[np.arange(n), a] = np.where(side == 1, hi[np.arange(n), a], lo[np.arange(n), a])
    d = np.where(rs.randint(0, 2, (n, 3)) == 1, np.float32(-0.0), np.float32(0.0)).astype(np.float32)
    b = np.where(rs.rand(n) < 0.7, (a + 1 + rs.randint(0, 2, n)) % 3, a)   # mostly along the plane, some across it
    d[np.arange(n), b] = np.where(rs.randint(0, 2, n) == 1, 1.0, -1.0)
    return _rays(o, d, tmin=0.0, tmax=np.inf)


def window_rays(rays, res):
    """every hit at t* re-fired with tmax in {t*, next(t*)} and tmin in {t*, prev(t*)}; and empty windows tmin = tmax = t*, tmin > tmax"""
    hit = res[:, 3] != MISS
    base, t = rays[hit], res[hit, 0].view(np.float32)
    out = []
    for tmin, tmax in ((None, t), (None, np.nextafter(t, np.float32(np.inf))), (t, None), (np.nextafter(t, np.float32(-np.inf)), None), (t, t), (t + 1, t)):
        r = base.copy()
        if tmin is not None: r[:, 3] = tmin
        if tmax is not None: r[:, 7] = tmax
        out.append(r)
    return np.concatenate(out) if out else np.zeros((0, 8), np.float32)


def bad_rays(wt, rs):
    """NaN and +-Inf in every component, zero directions: no hit anywhere"""
    c = wt.reshape(-1, 3).astype(np.float64).mean(0)
    base = _rays(np.tile((c + [0.1, 5.0, 0.2]).astype(np.float32), (1, 1)), np.array([[0.01, -1.0, 0.02]], np.float32))
    out = []
    for j in range(8):
        for val in (np.nan, np.inf, -np.inf):
            r = base.copy(); r[0, j] = val; out.append(r)
    z = base.copy(); z[0, 4:7] = 0.0; out.append(z)
    z = base.copy(); z[0, 4:7] = -0.0; out.append(z)
    return np.concatenate(out)


def grazing_rays(wt, rs, n):
    """in a triangle's plane, or tilted out of it by at most 1e-4 rad, through an interior point (ill-conditioned by construction)"""
    v = wt.reshape(-1, 3, 3).astype(np.float64)
    k = rs.randint(0, len(v), n)
    nrm = np.cross(v[k, 1] - v[k, 0], v[k, 2] - v[k, 0])
    ok = np.linalg.norm(nrm, axis=1) > 0
    k, nrm = k[ok], nrm[ok] / np.linalg.norm(nrm[ok], axis=1, keepdims=True)
    m = len(k)
    p = (rs.dirichlet((2, 2, 2), m)[:, :, None] * v[k]).sum(1)
    tan = np.cross(nrm, _unit(rs, m)); tan /= np.linalg.norm(tan, axis=1, keepdims=True)
    ang = np.where(rs.rand(m) < 0.3, 0.0, rs.uniform(-1e-4, 1e-4, m))
    d = np.cos(ang)[:, None] * tan + np.sin(ang)[:, None] * nrm
    scale = np.linalg.norm(v[k, 1] - v[k, 0], axis=1)[:, None]
    o = (p - d * scale * rs.uniform(0.5, 3.0, (m, 1))).astype(np.float32)
    return _rays(o, d.astype(np.float32))


def dyadic_rays():
    """straight down and straight up at every 1/8 point of the dyadic grid: vertices, edge midpoints, diagonals, interiors; t = 2 exactly"""
    g = np.arange(-1.125, 1.126, 0.125, dtype=np.float32)
    x, z = [a.ravel() for a in np.meshgrid(g, g, indexing="ij")]
    down = _rays(np.stack([x, np.full_like(x, 2.0), z], 1), np.tile(np.array([[0.0, -1.0, 0.0]], np.float32), (len(x), 1)))
    up = _rays(np.stack([x, np.full_like(x, -2.0), z], 1), np.tile(np.array([[-0.0, 1.0, 0.0]], np.float32), (len(x), 1)))
    return np.concatenate([down, up])


@functools.lru_cache(maxsize=None)
def ray_sets(name, refit=False, n=192):
    """{set name: (rays float32[n, 8], ill-conditioned by construction bool[n])}, from the emulator's structure of `name` (node planes: of
    the refitted structure when `refit`, and the brute-force hits the windows clip)"""
    emu = _emu()
    wt, _ = parity.world_triangles(scene(name))
    rs = np.random.RandomState(sum(map(ord, name)))
    w = make_world(emu, name, refit)
    sets = {}
    if name == "dyadic":
        sets["edges"] = dyadic_rays()
    else:
        sets["edges"] = edge_rays(wt, rs, per=max(8, n // 15))
        sets["interior"] = interior_rays(wt, rs, n)
        sets["planes"] = plane_rays(w.tlas_download(), rs, n)
    hits = w.trace_rays(sets["edges"], brute_force=True)
    sets["windows"] = window_rays(sets["edges"], hits)[: 6 * n]
    sets["bad"] = bad_rays(wt, rs)
    out = {k: (r, np.zeros(len(r), bool)) for k, r in sets.items()}
    if name != "dyadic":
        g = grazing_rays(wt, rs, n // 2)
        out["grazing"] = (g, np.ones(len(g), bool))
    w.close()
    return out


def _emu():
    from kajiya_b200._abi import KjbLib
    return KjbLib(conftest._ensure_built(conftest.EMU_SO, "build_emu"))


# ------------------------------------------------------------------------------------------------ checks
def check_walk_equals_brute_force(walk, brute, rays, ill, wt, mode, what):
    """exact on conditioned rays; on the others the walk's hit is a true hit no closer than the brute force's (and no invented hit)"""
    cond = conditioned(rays, brute, wt) & ~ill
    col = slice(3, 4) if mode["any_hit"] else slice(0, 4)
    bad = np.nonzero(cond & (walk[:, col] != brute[:, col]).any(1))[0]
    assert not len(bad), f"{what} {mode}: {len(bad)} of {int(cond.sum())} conditioned rays differ, e.g. ray {rays[bad[0]].tolist()} walk {walk[bad[0]].tolist()} brute {brute[bad[0]].tolist()}"
    wh, bh = walk[:, 3] != MISS, brute[:, 3] != MISS
    assert not (wh & ~bh).any(), f"{what} {mode}: the walk reports a hit the brute force does not have"
    if not mode["any_hit"]:
        both = ~cond & wh
        tw, tb = walk[both, 0].view(np.float32), brute[both, 0].view(np.float32)
        assert (tw >= tb).all() and ((tw > tb) | (walk[both, 3] >= brute[both, 3])).all(), f"{what} {mode}: the walk beat the brute force"
    return int(cond.sum()), int((~cond).sum())


def oracle_brute(oracle_lib, name, rays, mode):
    w = make_world(oracle_lib, name)
    out = np.zeros((len(rays), 4), np.uint32)
    r = np.ascontiguousarray(rays, np.float32)
    f = oracle_lib.dll.kjo_trace_rays
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_int, C.c_int, C.c_int, C.c_void_p]
    f(w.ctx, r.ctypes.data, len(r), 1, int(mode["any_hit"]), int(mode["cull_back"]), out.ctypes.data)
    w.close()
    return out


CPU_SCENES = ["cornell", "ruins", "atrium_20k", "cornell_far", "coincident", "ties", "dyadic"]


@pytest.mark.parametrize("refit", [False, True], ids=["rebuilt", "refitted"])
@pytest.mark.parametrize("name", CPU_SCENES)
def test_walk_equals_brute_force(emu_lib, oracle_lib, name, refit):
    """(a) walk == brute force on the product, and (b) the product's brute force == the oracle's, on every ray set, in all four modes"""
    if refit and name in ("coincident", "dyadic"):
        pytest.skip("one instance of a flat grid / the fallback tree: the refit is covered by the other scenes")
    wt, _ = parity.world_triangles(scene(name))
    w = make_world(emu_lib, name, refit=refit)
    assert w.tlas_stats() == dict(rebuilds=1, refits=int(refit))
    tree = w.tlas_download()
    v0, e1, e2 = tri_arrays(wt)
    recs = tree["tris"][np.argsort(tree["tris"][:, 3], kind="stable")][: len(wt)]
    assert np.array_equal(recs[:, 0:3].view(np.float32), v0.astype(np.float32)) and np.array_equal(recs[:, 4:7].view(np.float32), e1.astype(np.float32))
    sets = ray_sets(name, refit)
    rays = np.concatenate([r for r, _ in sets.values()]); ill = np.concatenate([i for _, i in sets.values()])
    nonfinite = np.isnan(rays).any(1) | ~np.isfinite(rays[:, [0, 1, 2, 4, 5, 6]]).all(1) | (rays[:, 4:7] == 0).all(1)
    counts = {}
    for mode in MODES:
        walk, brute = w.trace_rays(rays, **mode), w.trace_rays(rays, brute_force=True, **mode)
        counts[str(mode)] = check_walk_equals_brute_force(walk, brute, rays, ill, wt, mode, name)
        assert (walk[nonfinite, 3] == MISS).all() and (brute[nonfinite, 3] == MISS).all()
        if not refit:
            ob = oracle_brute(oracle_lib, name, rays, mode)
            col = slice(3, 4) if mode["any_hit"] else slice(0, 4)
            bad = np.nonzero((ob[:, col] != brute[:, col]).any(1))[0]
            assert not len(bad), f"{name} {mode}: product brute force != oracle brute force on {len(bad)} rays, e.g. {rays[bad[0]].tolist()}"
    assert (brute[:, 3] != MISS).mean() > 0.2   # the sets mostly hit
    w.close()


def test_tie_clusters_split_as_intended(emu_lib):
    """the tie scene really puts T's lowest copy and a higher copy in different leaves, and the higher one's leaf box is the wider"""
    w = make_world(emu_lib, "ties")
    tree = w.tlas_download()
    leaf_of = {}
    nodes = tree["nodes"]
    for i in range(len(nodes)):
        for k in range(2):
            ch = int(nodes[i, 12 + k].view(np.int32))
            if ch < 0:
                e = ~ch
                for g in tree["tris"][e >> 3:(e >> 3) + (e & 7) + 1, 3]:
                    leaf_of[int(g)] = (i, k)
    split = sum(leaf_of[8 * c] != leaf_of[8 * c + 4] for c in range(len(tree["tris"]) // 8))
    assert split == len(tree["tris"]) // 8
    res = w.trace_rays(ray_sets("ties")["interior"][0], brute_force=True)
    hit = res[:, 3] != MISS
    assert (res[hit, 3] % 8 == 0).mean() > 0.3   # many rays end on T, whose answer is a tie between copies 0..4 of a cluster
    w.close()


@np.errstate(all="ignore")   # NaN / Inf rays and degenerate triangles
def _ambiguous(rays, wt, cull_back, rel=1e-5):
    """rays whose float32 answer float64 cannot predict: a triangle within rounding of an edge or of the window inside the range that
    matters, a grazing winner, or a runner-up (other than an identical copy) within rel of the winner's t"""
    v0, e1, e2 = tri_arrays(wt)
    amb = np.zeros(len(rays), bool)
    for s in range(0, len(rays), 256):
        r = rays[s:s + 256]
        m = mt64(r, v0, e1, e2)
        tmin, tmax = r[:, 3:4].astype(np.float64), r[:, 7:8].astype(np.float64)
        marg = np.minimum(np.minimum(m["u"], m["v"]), 1 - m["u"] - m["v"])
        valid = np.isfinite(m["t"]) & (m["det"] != 0)
        if cull_back:   # a facing float32 could flip counts as a candidate
            valid &= (m["det"] > 0) | (m["cos"] <= 1e-3)
        inside = valid & (marg >= 0) & (m["t"] > tmin) & (m["t"] < tmax)
        t_hit = np.where(inside, m["t"], np.inf)
        t1 = t_hit.min(1)
        near = valid & (np.abs(marg) <= np.maximum(1e-5, m["bary_err"])) & (m["t"] > tmin - rel * np.abs(tmin) - 1e-30) & (m["t"] <= t1[:, None] * (1 + rel) + 1e-30)
        thr = np.maximum(1e-5, m["bary_err"])
        near |= valid & (marg >= -thr) & ((np.abs(m["t"] - tmin) <= rel * np.abs(m["t"])) | (np.abs(tmax - m["t"]) <= rel * np.abs(m["t"])))
        amb[s:s + 256] |= near.any(1)
        w = np.argmin(np.where(t_hit == t1[:, None], np.arange(t_hit.shape[1])[None], 1 << 40), axis=1)
        hasw = np.isfinite(t1)
        twin = (wt[None] == wt[w][:, None]).all(-1)
        runner = np.where(twin, np.inf, t_hit).min(1)
        at = lambda x: np.broadcast_to(x, m["t"].shape)[np.arange(len(r)), w]
        bound = t_error_bound({k: at(x) for k, x in m.items()}) * U   # origins close to a large triangle: t itself is not good to rel
        amb[s:s + 256] |= hasw & ((at(m["cos"]) <= 1e-3) | (runner <= t1 * (1 + rel)) | ~(bound <= rel / 2))
        amb[s:s + 256] |= np.isnan(r).any(1) | ~np.isfinite(r[:, [0, 1, 2, 4, 5, 6]]).all(1)
    return amb


@np.errstate(all="ignore")
def f64_reference(rays, wt, cull_back):
    """the contract evaluated in float64: inclusive edges, tmin < t < tmax, back faces det < 0, smallest t then smallest gid"""
    v0, e1, e2 = tri_arrays(wt)
    gid, t = np.full(len(rays), MISS, np.int64), np.zeros(len(rays))
    for s in range(0, len(rays), 256):
        r = rays[s:s + 256]
        m = mt64(r, v0, e1, e2)
        ok = np.isfinite(m["t"]) & (m["det"] != 0) & (m["u"] >= 0) & (m["v"] >= 0) & (m["u"] + m["v"] <= 1)
        ok &= (m["t"] > r[:, 3:4]) & (m["t"] < r[:, 7:8])
        if cull_back:
            ok &= m["det"] > 0
        th = np.where(ok, m["t"], np.inf)
        t1 = th.min(1)
        w = np.argmin(np.where(th == t1[:, None], np.arange(th.shape[1])[None], 1 << 40), axis=1)
        hit = np.isfinite(t1)
        gid[s:s + 256] = np.where(hit, w, MISS); t[s:s + 256] = np.where(hit, t1, 0)
    return gid, t


@pytest.mark.parametrize("name", ["cornell", "ruins", "cornell_far", "ties", "dyadic"])
def test_float64_reference(emu_lib, name):
    """(c) where float32 rounding cannot flip the answer: hit or miss, gid, t to 1e-5 relative; and on the dyadic grid (every float32
    operation exact) all of it exactly: inclusive shared edges and vertices resolved to the smaller gid, exclusive tmin / tmax.  Also
    the culling slack's error bound: float32's t is within the written bound of float64's on every conditioned hit."""
    wt, _ = parity.world_triangles(scene(name))
    w = make_world(emu_lib, name)
    sets = ray_sets(name)
    rays = np.concatenate([r for r, _ in sets.values()])
    checked = 0
    for cull in (False, True):
        res = w.trace_rays(rays, cull_back=cull)
        gid, t = f64_reference(rays, wt, cull)
        keep = np.ones(len(rays), bool) if name == "dyadic" else ~_ambiguous(rays, wt, cull)
        got_gid = res[:, 3].astype(np.int64)
        bad = np.nonzero(keep & (got_gid != gid))[0]
        assert not len(bad), f"{name} cull={cull}: {len(bad)} of {int(keep.sum())} rays: gid {got_gid[bad[:4]]} vs float64 {gid[bad[:4]]}, ray {rays[bad[0]].tolist()}"
        hit = keep & (gid != MISS)
        t32 = res[hit, 0].view(np.float32).astype(np.float64)
        if name == "dyadic":
            assert np.array_equal(t32, t[hit])
        else:
            rel = np.abs(t32 - t[hit]) / np.abs(t[hit])
            assert (rel <= 1e-5).all(), f"{name}: t off by {rel.max()} relative on ray {rays[hit][np.argmax(rel)].tolist()}"
        anyh = w.trace_rays(rays, any_hit=True, cull_back=cull)
        assert np.array_equal((anyh[keep, 3] != MISS), gid[keep] != MISS)
        # the slack covers Moeller-Trumbore's t error: measured against float64 on every hit within the limit
        h = res[:, 3] != MISS
        v0, e1, e2 = tri_arrays(wt)
        m = mt64(rays[h], v0, e1, e2, res[h, 3].astype(np.int64))
        b = t_error_bound({k: x[:, 0] for k, x in m.items()})
        err = np.abs(res[h, 0].view(np.float32).astype(np.float64) - m["t"][:, 0]) / np.abs(m["t"][:, 0]) / U
        within = np.isfinite(b) & (b <= 0.9 * SLACK_K - 6)
        assert (err[within] <= b[within]).all(), f"{name}: t error {err[within].max()} u over its bound"
        checked += int(keep.sum())
    if name == "dyadic":
        res = w.trace_rays(sets["edges"][0])
        assert (res[:, 3] != MISS).sum() == 2 * 17 * 17   # the 1/8 lattice over [-1.125, 1.125]: all but the outer ring hit, from both sides
    assert checked > 0.15 * 2 * len(rays)   # edge and window rays are ambiguous by design; interior and plane rays mostly are not
    w.close()


# ------------------------------------------------------------------------------------------------ GPU (H100)
def gpu_sets(wt, tree, seed, n=16384):
    rs = np.random.RandomState(seed)
    e = edge_rays(wt, rs, per=n // 30)
    return e, np.concatenate([interior_rays(wt, rs, n // 4), plane_rays(tree, rs, n // 8), bad_rays(wt, rs)]), grazing_rays(wt, rs, n // 16)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["atrium", "ruins"])
def test_gpu_walk_equals_brute_force(cuda_lib, name):
    """(a) on the H100: the full atrium (245 k triangles) and ruins (2.1 M), ~16 k rays per set, brute force over every triangle"""
    import time
    sc, view = scenes.atrium() if name == "atrium" else scenes.ruins()
    wt, _ = parity.world_triangles(sc)
    w = parity.make_world(cuda_lib, sc, 16, 8)
    w.render_frame(**view)
    t0 = time.perf_counter()
    edges, rest, graze = gpu_sets(wt, w.tlas_download(), 11)
    windows = window_rays(edges, w.trace_rays(edges, brute_force=True))
    rays = np.concatenate([edges, windows, rest, graze])
    ill = np.concatenate([np.zeros(len(rays) - len(graze), bool), np.ones(len(graze), bool)])
    for mode in MODES:
        check_walk_equals_brute_force(w.trace_rays(rays, **mode), w.trace_rays(rays, brute_force=True, **mode), rays, ill, wt, mode, name)
    print(f"[ray contract] {name}: {len(wt)} triangles, {len(rays)} rays x 4 modes, walk + brute force: {time.perf_counter() - t0:.1f} s")
    w.close()


@pytest.mark.gpu
@pytest.mark.parametrize("refit", [False, True], ids=["rebuilt", "refitted"])
def test_gpu_equals_the_emulator(cuda_lib, emu_lib, refit):
    """the nvcc build of the ray code (-fmad=false, explicit kjb_fma) returns the emulator's words bit for bit, walk and brute force"""
    for name in CPU_SCENES:
        if refit and name in ("coincident", "dyadic"):
            continue
        sets = ray_sets(name, refit)
        rays = np.concatenate([r for r, _ in sets.values()])
        wg, we = make_world(cuda_lib, name, refit), make_world(emu_lib, name, refit)
        for mode in MODES:
            for bf in (False, True):
                a, b = wg.trace_rays(rays, brute_force=bf, **mode), we.trace_rays(rays, brute_force=bf, **mode)
                bad = np.nonzero((a != b).any(1))[0]
                assert not len(bad), f"{name} {mode} brute_force={bf}: {len(bad)} rays differ, e.g. {rays[bad[0]].tolist()}: {a[bad[0]].tolist()} vs {b[bad[0]].tolist()}"
        wg.close(); we.close()
