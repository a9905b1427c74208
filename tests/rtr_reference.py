"""A float64 restatement of kajiya's reflection cleanup shader (`rtr/spatial_cleanup.hlsl`, R6 "reflection cleanup") and of the
unsigned 10- and 11-bit floats its R11G11B10 output is stored in, independent of the kernels and of the oracle.

Written from the HLSL and the Vulkan specification alone (cited as `file:line` and by section); nothing here comes from `oracle/`
or `kajiya_b200/csrc/`.  The rules are those of `taa_reference.py`, whose texel loads it reuses: continuous math in float64 on
exactly decoded texels, index and branch arithmetic (`filter_idx`, the sample count) in float32 as the HLSL writes it.
"""
import numpy as np

from taa_reference import F32, load, near_integer, pixel_grid, saturate

# ---------------------------------------------------------------- unsigned 11- and 10-bit floats (Vulkan specification, "Fundamentals":
# "Unsigned 11-Bit Floating-Point Numbers" and "Unsigned 10-Bit Floating-Point Numbers")
#
# Layout: 5 exponent bits E, then m = 6 (11-bit) or 5 (10-bit) mantissa bits M.  Value: E == 0 -> 2^-14 * M / 2^m; 0 < E < 31 ->
# 2^(E-15) * (1 + M / 2^m); E == 31, M == 0 -> +Inf; E == 31, M != 0 -> NaN.
# From float: finite values round to a representable finite value, and an implementation may always round towards zero (which is
# what R11G11B10 stores here); negative values and -Inf become 0; finite values above the largest finite (65024, 64512) become
# it; +Inf stays +Inf; every NaN becomes a positive NaN.
MAX_FINITE = {6: 65024.0, 5: 64512.0}


def uf_decode(code, m):
    """the value of unsigned small-float codes (int array), mantissa width m"""
    code = np.asarray(code, np.int64)
    e, mant = code >> m, code & ((1 << m) - 1)
    with np.errstate(invalid="ignore"):
        v = np.where(e == 0, np.ldexp(mant.astype(np.float64), -14 - m), np.ldexp(1.0 + mant / float(1 << m), e - 15))
        return np.where(e == 31, np.where(mant == 0, np.inf, np.nan), v)


def uf_encode_trunc(v, m):
    """float64 -> unsigned small-float code by the specification's rule, rounding towards zero; NaN -> the positive NaN with the
    top mantissa bit set"""
    v = np.asarray(v, np.float64)
    with np.errstate(invalid="ignore"):
        fin = np.isfinite(v) & (v > 0)
        x = np.where(fin, np.minimum(v, MAX_FINITE[m]), 1.0)
        fr, ex = np.frexp(x)                                       # x = fr * 2^ex, fr in [0.5, 1)
        e = ex - 1 + 15                                            # biased exponent of x
        normal = e >= 1
        mant_n = np.floor((fr * 2.0 - 1.0) * (1 << m)).astype(np.int64)
        mant_d = np.floor(np.ldexp(x, 14 + m)).astype(np.int64)    # E == 0: M = floor(x / 2^(-14-m))
        code = np.where(normal, (np.maximum(e, 1).astype(np.int64) << m) | mant_n, mant_d)
        code = np.where(fin, code, 0)
        code = np.where(v == np.inf, 31 << m, code)
        return np.where(np.isnan(v), (31 << m) | (1 << (m - 1)), code)


def r11g11b10_codes(word):
    w = np.asarray(word, np.uint32).astype(np.int64)
    return np.stack([w & 2047, (w >> 11) & 2047, (w >> 22) & 1023], axis=-1)


def a2r10g10b10_decode(word):
    """A2R10G10B10_UNORM_PACK32: R in bits 20-29, G in 10-19, B in 0-9, each / 1023"""
    w = np.asarray(word, np.uint32).astype(np.int64)
    return np.stack([(w >> 20) & 1023, (w >> 10) & 1023, w & 1023], axis=-1) / 1023.0


# ---------------------------------------------------------------- R6 "reflection cleanup": rtr/spatial_cleanup.hlsl
def spatial_cleanup(input_tex, depth, geometric_normal, offsets, view_to_clip_11, clip_to_view_43, frame_index, rows=None):
    """rtr/spatial_cleanup.hlsl:19-65 -> {"output_tex": (rgb value, slack)}, mask, stats.

    `input_tex` RGBA float64 (decoded f16), `depth` (H, W, 1), `geometric_normal` raw A2R10G10B10 words (H, W, 1), `offsets` the
    int4[512] constant table.  `slack` is how far a float32 evaluation may move the value before it is stored: 0 where the centre
    is stored as it is (:27-29); where the shader filters, 2^-20 of the value for the roundings of a positive weighted mean, plus
    its change under the float32 uncertainty of each weight (the depth term's exponent, and `dp^3` when `dp` is small) -- the
    `vsum / wsum` of :64.  The mask marks `filter_idx` arguments within reach of an integer; `center.w >= 8` and `< 4` compare an
    f16 value with a constant, and `8 - w / 2` is exact in float32 for every f16 `w` below 8, so neither they nor the sample
    count's truncation can flip."""
    H, W = input_tex.shape[:2]
    px, py = pixel_grid(W, H, rows)
    center = load(input_tex, px, py)                                  # :21
    cd = load(depth, px, py)[..., 0]                                  # :22
    csc = center[..., 3]                                              # :23
    through = (csc >= 8.0) | (cd == 0.0)                              # :27-29
    nc = load_normal(geometric_normal, px, py)                        # :32

    # :35-36 float32 as written: depth_to_view_z (inc/frame_constants.hlsl:192-194) = rcp(depth * -clip_to_view._43)
    d32 = np.where(through, F32(1.0), cd).astype(F32)
    vz = F32(1.0) / (d32 * -F32(clip_to_view_43))
    radius = F32(0.5) * F32(view_to_clip_11) / -vz
    fi_arg = radius * F32(7.0)
    filter_idx = np.clip(fi_arg, F32(0.0), F32(7.0)).astype(np.int64)
    radius64 = 0.5 * float(F32(view_to_clip_11)) * d32.astype(np.float64) * float(F32(clip_to_view_43))
    mask = ~through & near_integer(radius64 * 7.0) & (radius64 * 7.0 < 7.5)

    # :41 clamp(int(8 - w / 2), 2, 8) and :43 kernel_scale, in float32
    sc = np.clip(np.trunc(F32(8.0) - csc.astype(F32) / F32(2.0)), 2, 8).astype(np.int64)
    ks = np.where(csc < 4.0, 2, 1)
    q = (((px & 1) | (py & 1) * 2) + int(frame_index)) & 3            # :44 (SHUFFLE_SUBPIXELS)
    offs = np.asarray(offsets, np.int64).reshape(-1, 4)

    vsum, wsum, taps = 0.0, 0.0, []
    for i in range(8):                                                # :46
        on = i < sc
        o = offs[(q * 16 + i) + 64 * filter_idx]                       # :48
        sx, sy = px + ks * o[..., 0], py + ks * o[..., 1]
        neigh = np.sqrt(load(input_tex, sx, sy)[..., :3])             # :50 linear_rgb_to_crunched_rgb (inc/working_color_space.hlsl:22-24)
        sd = load(depth, sx, sy)[..., 0]                              # :51
        ns = load_normal(geometric_normal, sx, sy)                    # :52
        with np.errstate(divide="ignore", invalid="ignore"):
            rel = nc[..., 2] * (cd / sd - 1.0)
            w = np.exp2(-50.0 * np.abs(rel))                          # :56
        dp = saturate(np.sum(nc * ns, axis=-1))                       # :57
        w = np.where(on, w * dp * dp * dp, 0.0)                       # :58
        with np.errstate(invalid="ignore"):
            vsum = vsum + np.where(on[..., None], neigh * w[..., None], 0.0)   # :60 (samples past the count are never read)
        wsum = wsum + w
        # float32 uncertainty of this weight, relative: the exponent's rounding and a dot product near 0 (cubed)
        with np.errstate(divide="ignore", invalid="ignore"):
            u = 2.0 ** -20 + np.nan_to_num(50.0 * np.abs(nc[..., 2]) * np.abs(cd / sd) * 2.0 ** -21, posinf=0.0) + 3.0 * 2.0 ** -22 / dp
        taps.append((neigh, w, np.where(on, np.nan_to_num(u, posinf=0.0), 0.0)))
    with np.errstate(divide="ignore", invalid="ignore"):
        mean = vsum / wsum[..., None]                                 # :64
        move = sum(np.where((w * u > 0)[..., None], np.abs(n - mean) * (w * u)[..., None], 0.0) for n, w, u in taps) / wsum[..., None]
    # an Inf tap makes the sum Inf, or NaN (Inf * 0) where its weight is 0; a float64 weight below float32's normal range may be 0
    # in float32, so which of the two the shader gets is open there
    for n, w, _ in taps:
        mask = mask | (~through & ~np.isfinite(n).all(-1) & (w > 0) & (w < 2.0 ** -126))
    filtered = mean * mean                                            # crunched_rgb_to_linear_rgb (inc/working_color_space.hlsl:25-27)
    slack = 2.0 ** -20 * filtered + 2.0 * np.abs(mean) * move
    value = np.where(through[..., None], center[..., :3], filtered)
    slack = np.where(through[..., None] | ~np.isfinite(slack), 0.0, slack)   # an Inf or NaN result has no float32 neighbourhood
    stats = {"through": through, "filtered_nan": ~through & np.isnan(filtered).any(-1), "wsum_zero": ~through & (wsum == 0),
             "filter_idx": filter_idx, "sample_count": sc, "kernel_scale": ks}
    return {"output_tex": (value, slack)}, mask, stats


def load_normal(words, x, y):
    """`geometric_normal_tex[px] * 2 - 1` (spatial_cleanup.hlsl:32, :52): reads outside the image are 0 before the remap"""
    return a2r10g10b10_decode(load(words, x, y)[..., 0]) * 2.0 - 1.0
