"""The intersection contract is ours (the reference delegates to the Vulkan driver): validate the oracle's BVH walker
against brute force over all triangles — same t, u, v and triangle id, including tie-breaks — on random rays and on the hostile ray
sets of tests/test_ray_contract.py (edges from far away, exact ties across leaves, node planes, tmin / tmax windows, bad values, grazing)."""
import ctypes as C, numpy as np
import pytest
import parity
import test_ray_contract as rc
from kajiya_b200 import scenes


def _trace(lib, w, rays, brute, any_hit=False, cull_back=False):
    out = np.zeros((len(rays), 4), np.uint32)
    r = np.ascontiguousarray(rays, np.float32)
    f = lib.dll.kjo_trace_rays
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_int, C.c_int, C.c_int, C.c_void_p]
    f(w.ctx, r.ctypes.data, C.c_uint32(len(r)), int(brute), int(any_hit), int(cull_back), out.ctypes.data)
    return out


def _random_rays(n, seed):
    rs = np.random.RandomState(seed)
    rays = np.zeros((n, 8), np.float32)
    rays[:, 0:3] = rs.uniform(-3, 3, (n, 3)); rays[:, 3] = 0.0
    d = rs.randn(n, 3); rays[:, 4:7] = d / np.linalg.norm(d, axis=1, keepdims=True); rays[:, 7] = 1e4
    rays[: n // 8, 4:7] = np.round(rays[: n // 8, 4:7])   # axis-aligned rays hit shared edges/corners: exercises ties
    rays[: n // 8, 4] += (np.abs(rays[: n // 8, 4:7]).sum(1) == 0)
    return rays


def _check(lib, scene, rays, ill=None, wt=None):
    """walk == brute force in all four modes; rays beyond the culling slack's conditioning limit (or tagged ill-conditioned) get the weaker
    check of tests/test_ray_contract.py"""
    w = parity.make_world(lib, scene[0], 16, 16)
    w.render_frame(**scene[1])   # uploads geometry + builds the BVH
    wt = parity.world_triangles(scene[0])[0] if wt is None else wt
    ill = np.zeros(len(rays), bool) if ill is None else ill
    for mode in rc.MODES:
        walk, brute = _trace(lib, w, rays, False, **mode), _trace(lib, w, rays, True, **mode)
        rc.check_walk_equals_brute_force(walk, brute, rays, ill, wt, mode, "oracle")
    assert (_trace(lib, w, rays, True)[:, 3] != rc.MISS).mean() > 0.2


def test_bvh_vs_brute_force_cornell(oracle_lib):
    _check(oracle_lib, scenes.cornell_box(), _random_rays(4000, 0))


def test_bvh_vs_brute_force_atrium(oracle_lib):
    scene, view = scenes.atrium(target_tris=6000)
    _check(oracle_lib, (scene, view), _random_rays(1500, 1))


@pytest.mark.parametrize("name", rc.CPU_SCENES)
def test_bvh_vs_brute_force_hostile_rays(oracle_lib, name):
    sets = rc.ray_sets(name)
    rays = np.concatenate([r for r, _ in sets.values()]); ill = np.concatenate([i for _, i in sets.values()])
    _check(oracle_lib, (rc.scene(name), scenes.cornell_box()[1]), rays, ill)
