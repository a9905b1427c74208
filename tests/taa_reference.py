"""A float64 restatement of kajiya's seven TAA shaders, independent of the kernels and of the oracle.

Written from the HLSL alone (`assets/shaders/taa/*.hlsl` and the includes they use, cited as `file:line` below); nothing here
comes from `oracle/` or `kajiya_b200/csrc/`.  It is what the per-pass tests in `test_taa_reference.py` compare each backend with.

Rules that make it a statement of the shader rather than of the port:
  - continuous math (weights, colour transforms, Catmull-Rom, variances, blends) runs in float64 on exactly decoded texels;
  - index and branch arithmetic runs in float32 as the HLSL writes it (`uint2((px + 0.5) * scale)`, `get_uv`,
    `floor(uv * size + 1e-3)`, the `> 1.75` ratio test, the dilation test, `uv + reproj == saturate(uv + reproj)`);
  - `min`/`max` are fmin/fmax, `saturate(NaN) = 0`, division by zero is IEEE, loads outside the image return 0;
  - `SampleLevel` is clamp-to-edge bilinear (or nearest) in full precision.

Every pass returns `{output name: (value, scale)}` plus a "near a decision" mask of its grid.  `value` is float64 (H, W, C);
`scale` is the largest absolute contribution of one tap to that texel and channel, which bounds the cancellation a float32
evaluation may suffer.  The mask marks texels where a float64 quantity lies within 2^-16 relative of a threshold whose float32
evaluation could flip (a luma sign feeding `luma_cutoff / s.x`, the dilation test, a nearest-sampling or `floor` argument near
an integer).  Comparisons of exactly stored values (depth in the dilation argmax, history validity) cannot flip and are not masked.
"""
import numpy as np

F32 = np.float32
MARGIN = 2.0 ** -16


def f32(x):
    return np.asarray(x, dtype=np.float32)


# ---------------------------------------------------------------- texel decode (exact; f16 and R32F widen with astype)
def decode_snorm16(a):
    return np.maximum(np.asarray(a, dtype=np.int16).astype(np.float64) / 32767.0, -1.0)


# ---------------------------------------------------------------- HLSL intrinsics
def saturate(x):
    return np.fmin(np.fmax(x, 0.0), 1.0)          # fmax(NaN, 0) = 0: saturate(NaN) = 0


def lerp(a, b, t):
    return a + (b - a) * t


def smoothstep(e0, e1, x):
    t = saturate((x - e0) / (e1 - e0))
    return t * t * (3.0 - 2.0 * t)


def length(v):
    return np.sqrt(np.sum(v * v, axis=-1))


def max3(v):                                      # inc/math.hlsl:6-8
    return np.fmax(v[..., 0], np.fmax(v[..., 1], v[..., 2]))


# ---------------------------------------------------------------- image access
def load(img, x, y):
    """`tex[int2(x, y)]`: texel (..., C), 0 outside the image (the ABI's rule for out-of-range loads)."""
    H, W = img.shape[:2]
    ok = (x >= 0) & (x < W) & (y >= 0) & (y < H)
    v = img[np.clip(y, 0, H - 1), np.clip(x, 0, W - 1)]
    return np.where(ok[..., None], v, 0.0)


def sample_bilinear(img, u, v):
    """`SampleLevel(sampler_l?c, uv, 0)`: clamp-to-edge bilinear at normalised (u, v), float64 weights."""
    H, W = img.shape[:2]
    x = np.asarray(u, np.float64) * W - 0.5
    y = np.asarray(v, np.float64) * H - 0.5
    x0, y0 = np.floor(x), np.floor(y)
    fx, fy = (x - x0)[..., None], (y - y0)[..., None]
    x0, y0 = x0.astype(np.int64), y0.astype(np.int64)
    xa, xb = np.clip(x0, 0, W - 1), np.clip(x0 + 1, 0, W - 1)
    ya, yb = np.clip(y0, 0, H - 1), np.clip(y0 + 1, 0, H - 1)
    top = img[ya, xa] * (1 - fx) + img[ya, xb] * fx
    bot = img[yb, xa] * (1 - fx) + img[yb, xb] * fx
    return top * (1 - fy) + bot * fy


def sample_nearest(img, u, v):
    """`SampleLevel(sampler_nnc, uv, 0)`: the texel under (u, v), clamped; also the mask of arguments within reach of a texel edge."""
    H, W = img.shape[:2]
    x = np.asarray(u, np.float64) * W
    y = np.asarray(v, np.float64) * H
    near = near_integer(x) | near_integer(y)
    ix = np.clip(np.floor(x), 0, W - 1).astype(np.int64)
    iy = np.clip(np.floor(y), 0, H - 1).astype(np.int64)
    return img[iy, ix], near


def near_integer(x):
    """A `floor` argument within 1e-5 (or 4 float32 ulps, past 21) of an integer: a float32 evaluation could land on either side."""
    x = np.asarray(x, np.float64)
    return np.abs(x - np.round(x)) <= np.maximum(1e-5, 2.0 ** -21 * np.abs(x))


def pixel_grid(w, h, rows=None):
    """Pixel coordinates of rows [r0, r1) (all rows by default) of a w x h grid."""
    r0, r1 = rows if rows is not None else (0, h)
    py, px = np.mgrid[r0:r1, 0:w]
    return px.astype(np.int64), py.astype(np.int64)


def get_uv(px, py, tex_size):
    """inc/uv.hlsl:4-6 `(float2(pix) + 0.5) * texSize.zw`, in float32."""
    ts = f32(tex_size)
    return (px.astype(F32) + F32(0.5)) * ts[2], (py.astype(F32) + F32(0.5)) * ts[3]


def scaled_px(px, py, scale):
    """`uint2((px + 0.5) * scale)` in float32 (reproject_history.hlsl:45, taa.hlsl:109, unjitter_taa.hlsl:68)."""
    return (((px.astype(F32) + F32(0.5)) * scale[0]).astype(np.int64),
            ((py.astype(F32) + F32(0.5)) * scale[1]).astype(np.int64))


# ---------------------------------------------------------------- colour (inc/color/ycbcr.hlsl, taa/taa_common.hlsl)
_YCBCR = ((0.2126, 0.7152, 0.0722), (-0.1146, -0.3854, 0.5), (0.5, -0.4542, -0.0458))   # inc/color/ycbcr.hlsl:5
_RGB = ((1.0, 0.0, 1.5748), (1.0, -0.1873, -0.4681), (1.0, 1.8556, 0.0))                 # inc/color/ycbcr.hlsl:9


def _mul3(m, c):
    # written out term by term (not a BLAS product), so signed zeros survive as they do in `mul(float3x3, float3)`
    return np.stack([m[i][0] * c[..., 0] + m[i][1] * c[..., 1] + m[i][2] * c[..., 2] for i in range(3)], axis=-1)


def sRGB_to_YCbCr(c):          # inc/color/ycbcr.hlsl:4-6
    return _mul3(_YCBCR, c)


def YCbCr_to_sRGB(c):          # inc/color/ycbcr.hlsl:8-10
    return np.fmax(0.0, _mul3(_RGB, c))


def linear_to_perceptual(a):   # taa/taa_common.hlsl:7-25 (TAA_NONLINEARITY_TYPE 1)
    return np.sqrt(np.fmax(0.0, a))


def perceptual_to_linear(a):   # taa/taa_common.hlsl:27-46
    return a * a


def decode_rgb(v):             # taa/taa_common.hlsl:48-55 (TAA_COLOR_MAPPING_MODE 1)
    m = max3(v)[..., None]
    return v * linear_to_perceptual(m) / np.fmax(1e-20, m)


def encode_rgb(v):             # taa/taa_common.hlsl:57-64
    m = max3(v)[..., None]
    return v * perceptual_to_linear(m) / np.fmax(1e-20, m)


def _luma_terms(c):
    """|each term| of the YCbCr luma row: the scale its float32 sum rounds against."""
    return np.abs(0.2126 * c[..., 0]) + np.abs(0.7152 * c[..., 1]) + np.abs(0.0722 * c[..., 2])


def _near_zero(x, scale):
    """Nonzero but within 2^-16 of `scale` from 0: the sign float32 gives it may differ."""
    return (x != 0) & (np.abs(x) <= MARGIN * scale)


def luma_weight(cutoff, luma):
    """`pow(saturate(luma_cutoff / s.x), 8)` (taa/filter_input.hlsl:53, taa/filter_history.hlsl:37)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        return saturate(cutoff / luma) ** 8


# ---------------------------------------------------------------- inc/image.hlsl:84-150 image_sample_catmull_rom_approx (5 taps)
def catmull_rom_5tap(tex, uvx, uvy, tex_size_xy, remap):
    """`image_sample_catmull_rom_5tap` (inc/image.hlsl:165-170 -> 84-150, useCornerTaps = false) -> (value, largest tap contribution).

    `uvx, uvy` are the shader's float32 coordinates; the texel anchor `floor(samplePos - 0.5f) + 0.5f` is float32 as written,
    the weights and the bilinear taps are float64.  The spline is continuous across texel edges, so the floor needs no margin."""
    tsx, tsy = F32(tex_size_xy[0]), F32(tex_size_xy[1])
    spx, spy = uvx * tsx, uvy * tsy                                   # image.hlsl:90
    t1x = np.floor(spx - F32(0.5)) + F32(0.5)                        # image.hlsl:91
    t1y = np.floor(spy - F32(0.5)) + F32(0.5)
    fx = (spx - t1x).astype(np.float64)                              # image.hlsl:95
    fy = (spy - t1y).astype(np.float64)
    t1x, t1y = t1x.astype(np.float64), t1y.astype(np.float64)

    def weights(f):                                                   # image.hlsl:100-108
        w0 = f * (-0.5 + f * (1.0 - 0.5 * f))
        w1 = 1.0 + f * f * (-2.5 + 1.5 * f)
        w2 = f * (0.5 + f * (2.0 - 1.5 * f))
        w3 = f * f * (-0.5 + 0.5 * f)
        return w0, w1 + w2, w2 / (w1 + w2), w3

    w0x, w12x, o12x, w3x = weights(fx)
    w0y, w12y, o12y, w3y = weights(fy)
    W, H = float(tsx), float(tsy)
    p0x, p3x, p12x = (t1x - 1) / W, (t1x + 2) / W, (t1x + o12x) / W  # image.hlsl:111-117
    p0y, p3y, p12y = (t1y - 1) / H, (t1y + 2) / H, (t1y + o12y) / H
    taps = ((p12x, p0y, w12x * w0y), (p0x, p12y, w0x * w12y), (p12x, p12y, w12x * w12y),
            (p3x, p12y, w3x * w12y), (p12x, p3y, w12x * w3y))     # image.hlsl:125-139, corner taps off
    wsum = sum(t[2] for t in taps)                                    # image.hlsl:146
    acc, scale = 0.0, 0.0
    for u, v, w in taps:
        c0 = remap(sample_bilinear(tex, u, v))
        wn = (w / wsum)[..., None]
        acc = acc + c0 * wn
        scale = np.fmax(scale, np.abs(c0 * wn))
        # the sampler's float32 coordinate `u * size - 0.5` is only known to a few ulps; next to a texel 10^5 times brighter
        # that moves the tap far more than its rounding does, so the tap's change over +-4 ulps of its texel coordinate is
        # counted as a contribution of its own (scaled up by 2^11, since the bound takes 2^-11 of it)
        for eu, ev in _ulp_shifts(u, v, tex.shape):
            shift = np.abs((remap(sample_bilinear(tex, u + eu, v + ev)) - c0) * wn)
            scale = np.fmax(scale, 2.0 ** 11 * shift)
    return acc, scale


# ---------------------------------------------------------------- T1 "reproject taa": taa/reproject_history.hlsl
def reproject_history(history, reprojection, depth, input_tex_size, output_tex_size, pre_exposure_delta, rows=None):
    """taa/reproject_history.hlsl:38-129 on the output grid -> {"output_tex", "closest_velocity_output"}, mask.

    The wave: 8x8 groups anchored at pixel (0, 0), lane = x % 8 + 8 * (y % 4) (8x4 per wave); lanes past the image edge run the
    dilation test too.  `should_dilate |= lane ^ 2` then `|= lane ^ 16` (:80,:82) ORs the quad {l, l^2, l^16, l^18}."""
    OW, OH = int(output_tex_size[0]), int(output_tex_size[1])
    r0, r1 = rows if rows is not None else (0, OH)
    Wp, q0, q1 = -(-OW // 8) * 8, r0 & ~3, -(-r1 // 4) * 4           # the dispatch covers whole 8x8 groups: whole 8x4 waves
    px, py = pixel_grid(Wp, q1, (q0, q1))
    its, ots = f32(input_tex_size), f32(output_tex_size)
    scale = its[:2] / ots[:2]                                         # :44
    rx, ry = scaled_px(px, py, scale)                                 # :45
    uvx, uvy = get_uv(px, py, output_tex_size)                        # :47

    # :50-75 the velocity bounding box of the four diagonal neighbours and the dilation test, in float32 as written
    vs = [load(reprojection, rx + dx, ry + dy)[..., :2] for dx, dy in ((-1, -1), (1, -1), (-1, 1), (1, 1))]
    vmin64, vmax64 = vs[0], vs[0]
    for v in vs[1:]:
        vmin64, vmax64 = np.fmin(vmin64, v), np.fmax(vmax64, v)
    vmin, vmax = vmin64.astype(F32), vmax64.astype(F32)
    lhs = vmax - vmin
    rhs = F32(0.1) * np.fmax(its[2:], np.abs(vmax + vmin))
    test = lhs > rhs
    should = np.any(test, axis=-1)
    # margin: a component whose float64 difference sits within 2^-16 of its threshold, when no other component decides
    lhs64, rhs64 = vmax64 - vmin64, 0.1 * np.fmax(its[2:].astype(np.float64), np.abs(vmax64 + vmin64))
    near_c = np.abs(lhs64 - rhs64) <= MARGIN * np.fmax(np.abs(lhs64), rhs64)
    near = np.any(near_c, axis=-1) & ~np.any(test & ~near_c, axis=-1)

    def quad_or(s):                                                   # :80 lane ^ 2 (x ^ 2), :82 lane ^ 16 (y ^ 2 within the 4-row wave)
        s = s | s[:, np.arange(Wp) ^ 2]
        return s | s[np.arange(q1 - q0) ^ 2, :]

    firm = quad_or(should & ~near)
    should = quad_or(should)
    mask_dilate = quad_or(near) & ~firm

    # :94-104 depth argmax over the 3x3, scan order, strict `>`: the first of equal depths wins
    cx, cy = rx.copy(), ry.copy()
    best = load(depth, rx, ry)[..., 0]
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            d = load(depth, rx + dx, ry + dy)[..., 0]
            take = should & (d > best)
            best = np.where(take, d, best)
            cx, cy = np.where(take, rx + dx, cx), np.where(take, ry + dy, cy)

    reproj_xy64 = load(reprojection, cx, cy)[..., :2]                 # :107
    reproj_xy = reproj_xy64.astype(F32)
    hx, hy = uvx + reproj_xy[..., 0], uvy + reproj_xy[..., 1]        # :109 float32 add

    def remap(v):                                                     # :33-35 HistoryRemap
        return np.concatenate([decode_rgb(v[..., :3] * float(F32(pre_exposure_delta))), v[..., 3:4]], axis=-1)

    packed, pscale = catmull_rom_5tap(history, hx, hy, output_tex_size[:2], remap)   # :118-120
    out = np.concatenate([packed[..., :3], np.fmax(0.0, packed[..., 3:4])], axis=-1)  # :125-128
    crop = (slice(r0 - q0, r1 - q0), slice(0, OW))
    return ({"output_tex": (out[crop], pscale[crop]),
             "closest_velocity_output": (reproj_xy64[crop], np.zeros_like(reproj_xy64[crop]))},
            mask_dilate[crop])


# ---------------------------------------------------------------- T2 "taa filter input": taa/filter_input.hlsl
def _input_remap(v):                                                  # filter_input.hlsl:20-22, input_prob.hlsl:31-33, taa.hlsl:56-58
    return sRGB_to_YCbCr(decode_rgb(v[..., :3]))


def filter_input(input_tex, depth, rows=None):
    """taa/filter_input.hlsl:30-89 on the input grid -> {"output_tex", "dev_output_tex"}, mask."""
    H, W = input_tex.shape[:2]
    px, py = pixel_grid(W, H, rows)
    center_depth = load(depth, px, py)[..., 0]                        # :78
    taps = []
    for y in (-1, 0, 1):
        for x in (-1, 0, 1):
            raw = load(input_tex, px + x, py + y)
            s = _input_remap(raw)                                     # :47
            d = load(depth, px + x, py + y)[..., 0]                   # :49
            rel = np.abs(np.fmax(1e-20, center_depth) / np.fmax(1e-20, d) - 1.0)   # inc/math.hlsl:64-66
            w = np.exp2(-np.fmin(16.0, 200.0 * rel)) * np.exp(-0.8 * (x * x + y * y))   # :44,:51-52
            taps.append((s, w, _luma_terms(decode_rgb(raw[..., :3]))))

    def inner(cutoff):                                                # :30-74
        wsum, acc, ex, ex2, scale, near = 0.0, 0.0, 0.0, 0.0, 0.0, False
        for s, w, lterms in taps:
            wl = w * luma_weight(cutoff, s[..., 0])                   # :53
            wsum = wsum + wl
            acc = acc + s * wl[..., None]
            ex, ex2 = ex + s, ex2 + s * s
            near = near | _near_zero(s[..., 0], lterms)
        absacc = 0.0
        with np.errstate(divide="ignore", invalid="ignore"):
            mean = acc / wsum[..., None]                              # :64
            for s, w, _ in taps:
                c = s * (w * luma_weight(cutoff, s[..., 0]) / wsum)[..., None]
                scale = np.fmax(scale, np.abs(c))
                absacc = absacc + np.abs(c[..., 0])
        ex, ex2 = ex / 9.0, ex2 / 9.0
        var = np.fmax(0.0, ex2 - ex * ex)                             # :71
        return mean, var, np.nan_to_num(scale), ex2, near, absacc

    m1, var1, _, ex2, near1, abs1 = inner(1e10)                       # :81
    cutoff = m1[..., 0] * 1.001                                       # :85
    m2, _, scale2, _, near2, _ = inner(cutoff)
    # the second pass's cutoff is a weighted mean of lumas: near 0 against the sum of its |terms|, its sign may differ
    mask = near1 | near2 | _near_zero(cutoff, abs1)
    dev = np.sqrt(var1)                                               # :88
    # `ex2 - ex * ex` in float32 keeps up to ~9 roundings of E[s^2] (2^-20.8 E[s^2]) when it cancels, and the square root turns
    # that into up to 2^-10.4 sqrt(E[s^2]): the scale is 2 sqrt(E[s^2]) against the 2^-11 factor of the bound
    dev_scale = 2.0 * np.sqrt(ex2)
    return {"output_tex": (m2, scale2), "dev_output_tex": (dev, dev_scale)}, mask


# ---------------------------------------------------------------- T3 "taa filter history": taa/filter_history.hlsl
def filter_history_kernel_radius(input_tex_size, output_tex_size):
    """filter_history.hlsl:55: `input_tex_size.x / output_tex_size.x > 1.75` in float32 -> 2, else 1."""
    return 2 if f32(input_tex_size)[0] / f32(output_tex_size)[0] > F32(1.75) else 1


def filter_history(input_tex, input_tex_size, output_tex_size, rows=None):
    """taa/filter_history.hlsl:15-62 on the output grid (the TAA input extent) -> {"output_tex"}, mask."""
    W, H = int(output_tex_size[0]), int(output_tex_size[1])
    px, py = pixel_grid(W, H, rows)
    k = filter_history_kernel_radius(input_tex_size, output_tex_size)   # :55
    uvx, uvy = get_uv(px, py, output_tex_size)                        # :48
    its = f32(input_tex_size)
    ax, ay = uvx * its[0] + F32(1e-3), uvy * its[1] + F32(1e-3)       # :21 float32, then floor
    sx, sy = np.floor(ax).astype(np.int64), np.floor(ay).astype(np.int64)
    mask = near_integer(uvx.astype(np.float64) * float(its[0]) + 1e-3) | near_integer(uvy.astype(np.float64) * float(its[1]) + 1e-3)
    taps = []
    for y in range(-k, k + 1):
        for x in range(-k, k + 1):
            raw = load(input_tex, sx + x, sy + y)[..., :3]
            taps.append((sRGB_to_YCbCr(raw), np.exp(-(0.8 / (k * k)) * (x * x + y * y)), _luma_terms(raw)))   # :31,:33

    def fi(cutoff):                                                   # :15-45
        wsum, acc, near = 0.0, 0.0, False
        for s, dw, lterms in taps:
            w = dw * luma_weight(cutoff, s[..., 0])
            wsum, acc = wsum + w, acc + s * w[..., None]
            near = near | _near_zero(s[..., 0], lterms)
        with np.errstate(divide="ignore", invalid="ignore"):
            mean = acc / wsum[..., None]                              # :44: 0/0 = NaN when every luma weight is 0
            scale, absacc = 0.0, 0.0
            for s, dw, _ in taps:
                c = s * (dw * luma_weight(cutoff, s[..., 0]) / wsum)[..., None]
                scale = np.fmax(scale, np.abs(c))
                absacc = absacc + np.abs(c[..., 0])
        return mean, np.nan_to_num(scale), near, absacc

    m1, _, near1, abs1 = fi(1e10)                                     # :49
    cutoff = m1[..., 0] * 1.001                                       # :50
    m2, scale2, near2, _ = fi(cutoff)
    mask = mask | near1 | near2 | _near_zero(cutoff, abs1)            # the cutoff's sign, as for each luma
    return {"output_tex": (m2, scale2)}, mask


# ---------------------------------------------------------------- T4 "taa input prob": taa/input_prob.hlsl
def input_prob(filtered_input, filtered_input_dev, filtered_history, reprojection, smooth_var_history, velocity_history,
               input_tex_size, sample_offset_pixels, delta_time_seconds, rows=None):
    """taa/input_prob.hlsl:47-109 on the input grid -> {"output_tex"}, mask (nearest-sampling arguments at a texel edge).

    Tolerance scale: the probability `exp2(-|idiff^2 / var| - 1000 vdiff)` divides by a bilinearly sampled variance and
    multiplies a sampled velocity by 1000, so it is far more sensitive to where the sampler lands than to rounding.  A sampler
    coordinate is known to a few float32 ulps of `u * size`; the probability is evaluated again with both samples moved by
    +-4 ulps in x and in y, and its change, times 2^11, is the scale (with the value itself)."""
    W, H = int(input_tex_size[0]), int(input_tex_size[1])
    px, py = pixel_grid(W, H, rows)
    ivar = 0.0
    for y in (-1, 0, 1):
        for x in (-1, 0, 1):
            ivar = np.fmax(ivar, load(filtered_input_dev, px + 2 * x, py + 2 * y)[..., :3])   # :57-63
    ivar = ivar * ivar                                                # :64
    its, off = f32(input_tex_size), f32(sample_offset_pixels)
    iux = (px.astype(F32) + off[0]) * its[2]                          # :67 float32
    iuy = (py.astype(F32) + off[1]) * its[3]
    closest_history, mask = sample_nearest(filtered_history, iux, iuy)   # :69 sampler_nnc
    rp = load(reprojection, px, py)[..., :2].astype(F32)
    sux, suy = iux + rp[..., 0], iuy + rp[..., 1]                     # :70-71 float32 add
    taps = [(load(filtered_input, px + x, py + y)[..., :3], load(reprojection, px + x, py + y)[..., :2])
            for y in (-1, 0, 1) for x in (-1, 0, 1)]                  # :94,:97

    def prob_at(u, v):
        closest_smooth_var = sample_bilinear(smooth_var_history, u, v)[..., :3]                             # :70
        closest_vel = sample_bilinear(velocity_history, u, v)[..., :2] * float(F32(delta_time_seconds))     # :71
        combined_var = np.fmin(closest_smooth_var, ivar * 10.0)       # :76
        prob_max = 0.0
        for s, vel in taps:
            idiff = s - closest_history[..., :3]                      # :95
            vdiff = length((vel - closest_vel) / np.fmax(1.0, np.abs(vel + closest_vel)))   # :98
            prob = np.exp2(-1.0 * length(idiff * idiff / np.fmax(1e-6, combined_var)) - 1000.0 * vdiff)   # :100
            prob_max = np.fmax(prob_max, prob)                        # :102
        return prob_max[..., None]

    out = prob_at(sux, suy)
    scale = np.abs(out)
    for eu, ev in _ulp_shifts(sux, suy, smooth_var_history.shape):
        scale = np.fmax(scale, 2.0 ** 11 * np.abs(prob_at(sux + eu, suy + ev) - out))
    return {"output_tex": (out, scale)}, mask


def _ulp_shifts(u, v, shape):
    """Moves of a normalised sampler coordinate by 4 float32 ulps of its texel coordinate, in +-x and +-y."""
    H, W = shape[:2]
    eu = 2.0 ** -21 * (np.abs(np.asarray(u, np.float64)) * W + 1.0) / W
    ev = 2.0 ** -21 * (np.abs(np.asarray(v, np.float64)) * H + 1.0) / H
    return ((eu, 0.0), (-eu, 0.0), (0.0, ev), (0.0, -ev))


# ---------------------------------------------------------------- T5 "taa prob filter": taa/filter_prob.hlsl
def filter_prob(input_tex, rows=None):
    """taa/filter_prob.hlsl:5-17: the 3x3 max (centre included; out-of-range loads are 0) -> {"output_tex"}, mask."""
    H, W = input_tex.shape[:2]
    px, py = pixel_grid(W, H, rows)
    prob = load(input_tex, px, py)[..., :1]                           # :6
    for y in (-1, 0, 1):
        for x in (-1, 0, 1):
            prob = np.fmax(prob, load(input_tex, px + x, py + y)[..., :1])   # :11-12
    return {"output_tex": (prob, np.zeros_like(prob))}, np.zeros(px.shape, bool)


# ---------------------------------------------------------------- T6 "taa prob filter2": taa/filter_prob2.hlsl
def filter_prob2(input_tex, rows=None):
    """taa/filter_prob2.hlsl:7-27 -> {"output_tex"}, mask.

    Tolerance scale: the output is `-log2(mean of 25 squished taps) / 10`; a relative error e in one tap's term moves it by
    e * term / sum / (10 ln 2), so each tap's contribution is counted as `term / sum / (10 ln 2)`."""
    H, W = input_tex.shape[:2]
    px, py = pixel_grid(W, H, rows)
    terms = []
    for y in range(-2, 3):
        for x in range(-2, 3):
            p = load(input_tex, px + 2 * x, py + 2 * y)[..., 0]       # :16
            terms.append(np.exp2(-np.clip(10.0 * p, 0.0, 100.0)))     # inc/math.hlsl:69-71 exponential_squish
    total = np.sum(terms, axis=0)
    prob = np.fmax(0.0, -1.0 / 10.0 * np.log2(1e-30 + total / 25.0))   # :21, inc/math.hlsl:74-76 exponential_unsquish
    scale = np.max(terms, axis=0) / total / (10.0 * np.log(2.0))
    return {"output_tex": (prob[..., None], scale[..., None])}, np.zeros(px.shape, bool)


# ---------------------------------------------------------------- inc/unjitter_taa.hlsl:58-125
def sample_image_unjitter_taa(img, input_size_xy, px, py, output_size_xy, sample_offset_pixels, kernel_scale, k):
    """`sample_image_unjitter_taa` with the InputRemap of taa.hlsl:56-58 -> (color (RGBA), coverage, ex, ex2, scale of colour taps).

    The sample positions are pixel coordinates, evaluated in float32 as written up to the offset `src_sample_loc - dst_sample_loc`
    (:71-73, :92, :95): at 3840 pixels their rounding (2.4e-4 px) moves the Gaussian weights exp2(-10 d^2 scale) by ~5e-3
    relative, more than an f16 ulp of the result, so that rounding is part of what the shader computes.  The weights and sums
    from the offset on are float64."""
    isz = f32(input_size_xy)
    scale = isz / f32(output_size_xy)                                 # :66-67
    bx, by = scaled_px(px, py, scale)                                 # :68
    s64 = scale.astype(np.float64)
    off = f32(sample_offset_pixels)
    dstx, dsty = px.astype(F32) + F32(0.5), py.astype(F32) + F32(0.5)    # :71
    bslx = (bx.astype(F32) + F32(0.5) + off[0] * F32(1)) / scale[0]  # :72-73
    bsly = (by.astype(F32) + F32(0.5) + off[1] * F32(-1)) / scale[1]
    res, ex, ex2, dsum, wsum, absres = 0.0, 0.0, 0.0, 0.0, 0.0, 0.0
    for y in range(-k, k + 1):
        for x in range(-k, k + 1):
            raw = load(img, bx + x, by + y)
            col = np.concatenate([_input_remap(raw), np.ones(raw.shape[:-1] + (1,))], axis=-1)   # :94 remap(fetch), alpha 1
            ox = ((bslx + F32(x) / scale[0]) - dstx).astype(np.float64) * kernel_scale   # :92,:95
            oy = ((bsly + F32(y) / scale[1]) - dsty).astype(np.float64) * kernel_scale
            d2 = ox * ox + oy * oy                                    # :97
            dev_wt = np.exp2(-d2 * s64[0])                            # :101
            wt = np.exp2(-10.0 * d2 * s64[0])                         # :103
            res = res + col * wt[..., None]
            absres = absres + np.abs(col) * wt[..., None]
            wsum = wsum + wt
            ex = ex + col[..., :3] * dev_wt[..., None]
            ex2 = ex2 + col[..., :3] * col[..., :3] * dev_wt[..., None]
            dsum = dsum + dev_wt
    return res, wsum, ex / dsum[..., None], ex2 / dsum[..., None], absres


# ---------------------------------------------------------------- T7 "taa": taa/taa.hlsl
def taa(input_tex, history, reprojection, closest_velocity, velocity_history, smooth_var_history, input_prob_tex,
        input_tex_size, output_tex_size, sample_offset_pixels, delta_time_seconds, rows=None):
    """taa/taa.hlsl:94-338 on the output grid -> {"temporal_output_tex", "output_tex", "smooth_var_output_tex",
    "velocity_output_tex"}, mask.

    Tolerance scale.  The result is `(clamped_history * history_coverage + center) / total_coverage` in YCbCr (:311), taken to
    RGB (:324) and squared by `encode_rgb` (:325): its scale is the absolute YCbCr contributions of the two terms (the centre's
    as the sum of its taps' |contributions|) through |YCbCr_to_sRGB|, doubled times the largest channel for the square.
    One quantity is worse conditioned than its taps: the variance `ex2 - ex^2` (:169), which cancels in flat neighbourhoods.
    Evaluated in float32 it keeps the roundings of two 9-tap weighted means and a square, up to ~30 * 2^-24 E[s^2] < 2^-18 E[s^2];
    the box it opens (:201-202), the clamp direction (:257) and the detail ratio over its 1e-3 floor (:235) pass that on to the
    colour and to the coverage (:280-282).  And the previous variance and velocity are bilinear samples whose coordinate is known
    to a few float32 ulps (see `input_prob`).  So the blend is evaluated again with the variance moved by 2^-18 E[s^2] (all
    channels up, all down, each channel up alone) and with the sampler coordinate moved by +-4 ulps in x and in y, and the change
    of each output, times 2^11, joins its scale."""
    OW, OH = int(output_tex_size[0]), int(output_tex_size[1])
    px, py = pixel_grid(OW, OH, rows)
    its, ots = f32(input_tex_size), f32(output_tex_size)
    frac = its[:2] / ots[:2]                                          # :108
    rx, ry = scaled_px(px, py, frac)                                  # :109
    uvx, uvy = get_uv(px, py, output_tex_size)                        # :118
    hp = load(history, px, py)[..., :4]                               # :120-122
    hist = hp[..., :3]
    hcov = np.fmax(0.0, hp[..., 3])

    csum, wsum = 0.0, 0.0                                             # :61-81 fetch_blurred_history(px, 2, 1)
    for y in range(-2, 3):
        for x in range(-2, 3):
            w = np.exp(-float(x * x + y * y))
            csum = csum + load(history, px + x, py + y)[..., :4] * w
            wsum = wsum + w
    bpacked = csum / wsum
    bhist = bpacked[..., :3]
    bcov = bpacked[..., 3:4]
    hist_y = sRGB_to_YCbCr(hist)                                      # :128-129
    bhist_y = sRGB_to_YCbCr(bhist)
    reproj = load(reprojection, rx, ry)                               # :131
    cv64 = load(closest_velocity, px, py)[..., :2]                    # :132
    cv = cv64.astype(F32)
    off = sample_offset_pixels
    csample = sample_image_unjitter_taa(input_tex, input_tex_size[:2], px, py, output_tex_size[:2], off, 1.0, 1)   # :134-141
    bsample = sample_image_unjitter_taa(input_tex, input_tex_size[:2], px, py, output_tex_size[:2], off, float(F32(0.333)), 1)
    center = csample[0][..., :3]                                      # :154-155
    coverage = csample[1]
    center_abs = csample[4][..., :3]
    bcenter = bsample[0][..., :3] / bsample[1][..., None]             # :160
    history_y = lerp(hist_y, bcenter, saturate(1.0 - hcov)[..., None])   # :162
    bhistory_y = lerp(bhist_y, bcenter, saturate(1.0 - bcov))        # :163
    iprob = load(input_prob_tex, rx, ry)[..., 0]                      # :165
    ex, ex2 = csample[2], csample[3]                                  # :167-169
    sx, sy = uvx + cv[..., 0], uvy + cv[..., 1]                       # :171,:175 float32 add
    dt = float(F32(delta_time_seconds))
    vel_now = cv64 / dt                                               # :174

    def sampled(u, v):
        prev_var = sample_bilinear(smooth_var_history, u, v)[..., 0:1]   # :171
        vel_prev = sample_bilinear(velocity_history, u, v)[..., :2]   # :175
        vel_diff = length((vel_now - vel_prev) / np.fmax(1.0, np.abs(vel_now + vel_prev)))   # :176
        return prev_var, saturate(0.3 + 0.7 * (1.0 - reproj[..., 2]) + vel_diff)   # :177
    box = lerp(0.8, 3.0, iprob)[..., None]                           # :194-199
    valid = (sx == np.fmin(np.fmax(sx, F32(0)), F32(1))) & (sy == np.fmin(np.fmax(sy, F32(0)), F32(1)))   # :224 float32
    v3 = valid[..., None]
    max_cov = np.fmax(2.0, 8.0 / (float(frac[0]) * float(frac[1])))   # :313

    def blend(var, prev_var, var_blend):                              # :169-331 from the neighbourhood variance on
        smooth_var = np.fmax(var, lerp(prev_var, var, var_blend[..., None]))   # :179
        smooth_var = lerp(var, smooth_var, saturate(iprob)[..., None])   # :181-182
        dev = np.sqrt(var)                                            # :184
        nmin, nmax = ex - dev * box, ex + dev * box                   # :201-202
        cbh = np.fmin(np.fmax(bhistory_y, nmin), nmax)                # :206
        clamping_event = length(np.fmax(0.0, np.fmax(bhistory_y - nmax, nmin - bhistory_y)) / np.fmax(0.01, ex))   # :211
        outlier3 = np.fmax(0.0, np.fmax(nmin - history_y, history_y - nmax) / (0.1 + np.fmax(np.fmax(np.abs(history_y), np.abs(ex)), 1e-5)))
        boutlier3 = np.fmax(0.0, np.fmax(nmin - bhistory_y, bhistory_y - nmax) / (0.1 + np.fmax(np.fmax(np.abs(bhistory_y), np.abs(ex)), 1e-5)))
        outlier, boutlier = max3(outlier3), max3(boutlier3)           # :217,:221
        ndo = np.fmax(0.0, outlier - boutlier) * 10.0                 # :228
        uhd = history_y - cbh                                         # :231
        tcd = np.abs(uhd[..., 0] / np.fmax(1e-3, dev[..., 0])) * 0.05   # :235
        allow = (saturate(ndo) * saturate(1.0 - tcd))[..., None]      # :239-242
        hd = lerp(history_y - bhistory_y, uhd, allow)                 # :251-254
        a, b = cbh - bhistory_y, bcenter - bhistory_y
        with np.errstate(invalid="ignore"):
            ibc = saturate(np.sum(a * b, axis=-1) / np.fmax(1e-5, length(a) * length(b)))   # :257-259
        keep = 1.0 - saturate(ibc)[..., None] * (1.0 - allow)         # :262-266
        ch_valid = cbh + hd * keep                                    # :267-270
        hcov_valid = hcov
        if frac[0] < F32(1.0):                                        # :274 float32
            hcov_valid = hcov * lerp(lerp(0.0, 0.9, keep[..., 0]), 1.0, saturate(10.0 * clamping_event))   # :280-282
        clamped_history = np.where(v3, ch_valid, cbh)                 # :286
        cov = np.where(valid, coverage, 1.0)                          # :287
        ctr = np.where(v3, center, bcenter)                           # :288
        hcov_out = np.where(valid, hcov_valid, 0.0)                   # :289
        clamped_history = lerp(clamped_history, history_y, smoothstep(0.5, 1.0, iprob)[..., None])   # :297-301
        total = np.fmax(1e-5, hcov_out + cov)                         # :310
        tr = (clamped_history * hcov_out[..., None] + ctr) / total[..., None]   # :311
        rgb = np.fmax(0.0, encode_rgb(YCbCr_to_sRGB(tr)))             # :324-326
        contrib = (np.abs(clamped_history) * hcov_out[..., None] + np.where(v3, center_abs, np.abs(bcenter))) / total[..., None]
        return rgb, np.fmin(max_cov, total), smooth_var, tr, contrib  # :315-317

    var = np.fmax(0.0, ex2 - ex * ex)                                 # :169
    prev_var, var_blend = sampled(sx, sy)
    rgb, total, smooth_var, tr, contrib = blend(var, prev_var, var_blend)
    # tolerance scale (see the docstring): the YCbCr contributions through |YCbCr_to_sRGB| and the square of encode_rgb, plus how far
    # the result moves when the variance carries the float32 residue of its cancellation
    gain = 2.0 * max3(np.fmax(0.0, _mul3(_RGB, tr)))[..., None]
    rgb_scale = _mul3(tuple(tuple(abs(c) for c in row) for row in _RGB), contrib) * gain
    cov_scale = np.zeros_like(total)
    # the smoothed variance is a blend of `var` and the sampled `prev_var` (:179-182); the float32 residue of `var`'s cancellation
    # is the variance move of the loop below
    sv_scale = np.fmax(np.abs(smooth_var), np.abs(prev_var))
    eps = 2.0 ** -18 * np.abs(ex2)
    signs = [(1.0, 1.0, 1.0), (-1.0, -1.0, -1.0), (1.0, 0.0, 0.0), (0.0, 1.0, 0.0), (0.0, 0.0, 1.0)]
    moved = [(np.fmax(0.0, var + np.array(sign) * eps), prev_var, var_blend) for sign in signs]
    moved += [(var,) + sampled(sx + eu, sy + ev) for eu, ev in _ulp_shifts(sx, sy, smooth_var_history.shape)]
    for args in moved:
        rgb_e, total_e, sv_e, _, _ = blend(*args)
        with np.errstate(invalid="ignore"):
            rgb_scale = np.fmax(rgb_scale, 2.0 ** 11 * np.nan_to_num(np.abs(rgb_e - rgb)))
        cov_scale = np.fmax(cov_scale, 2.0 ** 11 * np.abs(total_e - total))
        sv_scale = np.fmax(sv_scale, 2.0 ** 11 * np.abs(sv_e - smooth_var))

    zeros1 = np.zeros(rgb.shape[:-1] + (1,))
    temporal = np.concatenate([rgb, total[..., None]], axis=-1)       # :330
    temporal_scale = np.concatenate([rgb_scale, cov_scale[..., None]], axis=-1)
    output = np.concatenate([rgb, zeros1], axis=-1)                   # :328,:331 this_frame_result.a stays 0
    output_scale = np.concatenate([rgb_scale, zeros1], axis=-1)
    return ({"temporal_output_tex": (temporal, temporal_scale), "output_tex": (output, output_scale),
             "smooth_var_output_tex": (smooth_var, sv_scale), "velocity_output_tex": (vel_now, np.zeros_like(vel_now))},
            np.zeros(px.shape, bool))
