"""A numpy restatement of the frame driver's camera: the matrices of camera.rs:71-125, the Halton jitter of world_renderer.rs:425-428
and the view block prepare_frame_constants builds from them (world_renderer.rs:1001-1108), in float32 as the Rust writes it.

`test_host_mirror.py` checks it against the frame constants the driver uploads; the per-pass reference tests build their view block
with it (`pass_harness.view_constants`)."""
import numpy as np


def halton(i, base):   # radical_inverse, world_renderer.rs:1116-1129 (float arithmetic as written there)
    val, inv_base = np.float32(0), np.float32(1) / np.float32(base)
    inv_bi = inv_base
    n = int(i)
    while n > 0:
        d = n % base
        val = np.float32(val + np.float32(d) * inv_bi)
        n = int(np.float32(n) * inv_base)
        inv_bi = np.float32(inv_bi * inv_base)
    return val


def quat_to_mat(q):
    x, y, z, w = [np.float32(v) for v in q]
    x2, y2, z2 = x + x, y + y, z + z
    xx, xy, xz, yy, yz, zz, wx, wy, wz = x * x2, x * y2, x * z2, y * y2, y * z2, z * z2, w * x2, w * y2, w * z2
    m = np.eye(4, dtype=np.float32)
    m[:3, 0] = [1 - (yy + zz), xy + wz, xz - wy]; m[:3, 1] = [xy - wz, 1 - (xx + zz), yz + wx]; m[:3, 2] = [xz + wy, yz - wx, 1 - (xx + yy)]
    return m


def mat4_mul(a, b):   # glam Mat4 * Mat4 in f32: each element accumulated in k order
    r = np.zeros((4, 4), np.float32)
    for c in range(4):
        for rr in range(4):
            s = np.float32(0)
            for k in range(4):
                s = np.float32(s + np.float32(a[rr, k] * b[k, c]))
            r[rr, c] = s
    return r


def camera(pos, rot, W, H, fov_deg=52.0, znear=0.01):   # camera.rs:71-125: infinite reverse-Z perspective
    T = np.eye(4, dtype=np.float32); T[:3, 3] = pos
    Ti = np.eye(4, dtype=np.float32); Ti[:3, 3] = [-p for p in pos]
    R, Ri = quat_to_mat(rot), quat_to_mat([-rot[0], -rot[1], -rot[2], rot[3]])
    view_to_world, world_to_view = mat4_mul(T, R), mat4_mul(Ri, Ti)
    fov = np.float32(fov_deg) * (np.float32(np.pi) / np.float32(180.0))             # f32::to_radians
    half = float(np.float32(0.5) * fov)
    h = np.float32(np.float32(np.cos(half)) / np.float32(np.sin(half)))               # f32 cos / sin (evaluated in f64 and rounded: within an ulp of any libm)
    ww = np.float32(h / (np.float32(W) / np.float32(H)))
    v2c = np.zeros((4, 4), np.float32); v2c[0, 0] = ww; v2c[1, 1] = h; v2c[3, 2] = -1; v2c[2, 3] = znear
    c2v = np.zeros((4, 4), np.float32); c2v[0, 0] = np.float32(1) / ww; c2v[1, 1] = np.float32(1) / h; c2v[2, 3] = -1; c2v[3, 2] = np.float32(1) / np.float32(znear)
    return dict(view_to_clip=v2c, clip_to_view=c2v, world_to_view=world_to_view, view_to_world=view_to_world)


def view_block(cam, prev, frame, W, H):
    """The 11 matrices of the view constants for frame `frame` of a W x H render (`cam`, `prev`: `camera()` of this frame and the
    previous one) -> ({name: 4x4 [row, col]}, sample_offset_pixels, sample_offset_clip)."""
    i = (frame % 128) + 1
    off = np.array([halton(i, 2) - np.float32(0.5), halton(i, 3) - np.float32(0.5)], np.float32)   # Halton(2,3) - 0.5 (world_renderer.rs:425-428)
    off_clip = np.array([np.float32(2.0) * off[0] / np.float32(W), np.float32(2.0) * off[1] / np.float32(H)], np.float32)
    J = np.eye(4, dtype=np.float32); J[0, 3], J[1, 3] = -off_clip[0], -off_clip[1]
    Ji = np.eye(4, dtype=np.float32); Ji[0, 3], Ji[1, 3] = off_clip[0], off_clip[1]
    v = dict(cam)
    v["view_to_sample"] = mat4_mul(J, cam["view_to_clip"]); v["sample_to_view"] = mat4_mul(cam["clip_to_view"], Ji)
    v["clip_to_prev_clip"] = mat4_mul(mat4_mul(mat4_mul(prev["view_to_clip"], prev["world_to_view"]), cam["view_to_world"]), cam["clip_to_view"])
    v["prev_view_to_prev_clip"], v["prev_clip_to_prev_view"] = prev["view_to_clip"], prev["clip_to_view"]
    v["prev_world_to_prev_view"], v["prev_view_to_prev_world"] = prev["world_to_view"], prev["view_to_world"]
    return v, off, off_clip
