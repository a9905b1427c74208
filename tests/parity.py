"""Shared parity harness: run the same frame sequence through two implementations of the C-ABI and compare
EVERY live image after every frame.  Integer images must match bit-for-bit; float images are compared on their
stored bits too (the numeric contract makes that possible) with a tolerance fallback reported separately."""
import numpy as np
from kajiya_b200.world import World
from kajiya_b200 import scenes
from kajiya_b200._abi import FMT_NAME

INT_FORMATS = {"RG32_UINT", "RGBA32_UINT", "R32_UINT"}


def make_world(lib, scene, width, height, **kw):
    w = World(lib, width, height, **kw)
    scenes.populate(w, scene)
    return w


def glossy(scene):
    """the Cornell box with glossy walls, so that the reflection passes really trace (roughness <= 0.6)"""
    import copy
    s = copy.deepcopy(scene)
    for i, m in enumerate(s[0][0]["materials"]):
        m["roughness"] = [0.05, 0.2, 0.35, 0.5, 0.8][i % 5]; m["metallic"] = [1.0, 0.0, 0.5][i % 3]
    return s


def world_triangles(scene):
    """gid-ordered (instance-major, as scenes.populate adds them) world-space triangles float32[n, 9] and tri_info uint32[n, 2], with the
    library's xform_point: ((m0 x + m1 y) + m2 z) + m3 in float32, no contraction"""
    tris, info, inst = [], [], 0
    for mesh, transforms in scene:
        p = np.asarray(mesh["positions"], np.float32)[np.asarray(mesh["indices"], np.int64)]
        for t in transforms:
            m = np.asarray(t, np.float32).reshape(12)
            w = np.empty_like(p)
            for r in range(3):
                w[:, r] = ((m[4 * r] * p[:, 0] + m[4 * r + 1] * p[:, 1]) + m[4 * r + 2] * p[:, 2]) + m[4 * r + 3]
            tris.append(w.reshape(-1, 9))
            n = len(w) // 3
            info.append(np.stack([np.full(n, inst, np.uint32), np.arange(n, dtype=np.uint32)], 1))
            inst += 1
    if not tris:
        return np.zeros((0, 9), np.float32), np.zeros((0, 2), np.uint32)
    return np.ascontiguousarray(np.concatenate(tris)), np.concatenate(info)


def compare_images(wa, wb, names=None, rtol=0.0):
    """returns list of (name, n_mismatching_texels, max_abs_err) for images that differ"""
    bad = []
    names = names or sorted(set(wa.image_names()) & set(wb.image_names()))
    for n in names:
        a, b = wa.image(n), wb.image(n)
        if a.shape != b.shape:
            bad.append((n, -1, float("inf"))); continue
        ra, rb = a.view(np.uint8).reshape(a.shape[0], a.shape[1], -1), b.view(np.uint8).reshape(b.shape[0], b.shape[1], -1)
        diff = (ra != rb).any(-1)
        if diff.any():
            fmt = FMT_NAME[wa.image_handle(n).format]
            if a.dtype.kind == "f":
                fa, fb = a.astype(np.float64), b.astype(np.float64)
                both_nan = np.isnan(fa) & np.isnan(fb)
                err = np.where(both_nan, 0.0, np.abs(fa - fb))
                mx = float(np.nanmax(err)) if err.size else 0.0
                if not np.isfinite(mx): mx = float("inf")
                # -0.0 vs +0.0 and NaN payloads are bit differences without numeric meaning
                num_diff = int((err > rtol * np.maximum(np.abs(fa), np.abs(fb))).any(-1).sum()) if rtol > 0 else int((err > 0).any(-1).sum())
                if num_diff:
                    bad.append((f"{n} [{fmt}]", num_diff, mx))
            else:
                bad.append((f"{n} [{fmt}]", int(diff.sum()), float(np.abs(a.astype(np.int64) - b.astype(np.int64)).max())))
    return bad


def run_lockstep(lib_a, lib_b, scene, view, width, height, frames, **kw):
    wa, wb = make_world(lib_a, scene, width, height, **kw), make_world(lib_b, scene, width, height, **kw)
    report = []
    for f in range(frames):
        wa.render_frame(**view); wb.render_frame(**view)
        bad = compare_images(wa, wb)
        report.append(bad)
    return wa, wb, report
