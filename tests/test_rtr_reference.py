"""R6 "reflection cleanup" against `rtr_reference.py`, a float64 restatement of kajiya's `rtr/spatial_cleanup.hlsl` that shares
nothing with the kernels or the oracle, and the R11G11B10 encoder the pass stores through, against the Vulkan specification.

The pass is driven alone through the C-ABI (`pass_harness.py`) on the oracle and the emulator, and on the H100.  Its output is
R11G11B10, stored by truncation, so the check is one-sided: each channel's code must lie between the codes of the reference value
minus and plus its float32 slack -- at most one ulp of the 6- or 5-bit mantissa below the value, none above.  Texels whose
`filter_idx` argument is within reach of an integer are excluded, counted and kept under 1 %.

The encoder keeps one documented departure from the specification (DESIGN §8): NaN stores as 0 and +Inf as the largest finite
value.  The exhaustive test pins exactly that and nothing else, for all 65 536 f16 codes in each channel.
"""
import numpy as np
import pytest

import rtr_reference as ref
from pass_harness import F16, DEPTH, R11G11B10, A2R10G10B10, Runners, frame_constants, view_constants

PASSES = {"cleanup": ("kjb_pass_rtr_cleanup", ["input_tex", "depth_tex", "geometric_normal_tex", "output_tex"], 0, ["spatial_resolve_offsets"])}


def offsets():
    from kajiya_b200 import scenes
    return scenes.spatial_resolve_offsets()


@pytest.fixture(scope="module")
def runners():
    rs = Runners(PASSES)
    yield rs
    rs.close()


@pytest.fixture(scope="module")
def cpu_runners(runners, oracle_lib, emu_lib):
    return [runners(oracle_lib), runners(emu_lib)]


@pytest.fixture(scope="module")
def gpu_runner(runners, cuda_lib):
    return runners(cuda_lib)


# ---------------------------------------------------------------- the product's rule: the specification's, but for two inputs
def product_codes(v, m):
    """the codes R11G11B10 stores for float64 values: the specification's round-towards-zero rule (`rtr_reference.uf_encode_trunc`),
    except NaN -> 0 and +Inf -> the largest finite code (DESIGN §8)"""
    v = np.asarray(v, np.float64)
    c = ref.uf_encode_trunc(v, m)
    c = np.where(np.isnan(v), 0, c)
    return np.where(v == np.inf, ref.uf_encode_trunc(ref.MAX_FINITE[m], m), c)


MBITS = (6, 6, 5)


# ---------------------------------------------------------------- seeded synthetic inputs
def case_cleanup(seed, w, h, frame_index, hostile=True):
    """RGBA16F reflections with sample counts (alpha) on both sides of 4 and 8 and at them; depths that put `filter_idx` on all of
    0-7, exact ties and sky; geometric normals that are smooth, flipped (zero weight), or near the zero vector; with `hostile`, also
    f16 subnormals, 6e4, +Inf and NaN texels, and +Inf beside sky, where the shader's weighted sum is Inf * 0."""
    rng = np.random.default_rng(seed)
    c = np.exp(rng.uniform(np.log(1e-4), np.log(3e2), (h, w, 4)))
    c[..., 3] = rng.choice([0.0, 0.5, 1.0, 2.0, 3.0, 3.5, 3.998, 4.0, 5.0, 7.0, 7.996, 8.0, 9.0, 16.0, 17.0], (h, w))
    spread = rng.uniform(size=(h, w)) < 0.3
    c[spread, 3] = rng.uniform(0.0, 10.0, np.sum(spread))
    pick = rng.uniform(size=(h, w))
    c[pick < 0.03, :3] = 0.0
    if hostile:
        c[(pick >= 0.03) & (pick < 0.05), :3] = rng.choice([6e-8, 3e-6, 5.9e-5], (np.sum((pick >= 0.03) & (pick < 0.05)), 3))
        c[(pick >= 0.05) & (pick < 0.06), :3] = rng.uniform(3e4, 6e4, (np.sum((pick >= 0.05) & (pick < 0.06)), 3))
        c[(pick >= 0.06) & (pick < 0.065), rng.integers(0, 3)] = np.inf
        c[(pick >= 0.065) & (pick < 0.067), rng.integers(0, 3)] = np.nan
    img = c.astype(np.float16)

    d = rng.choice(np.float32([0.002, 0.005, 0.0031, 0.009]), (h, w)).astype(np.float32)   # ties
    noisy = rng.uniform(size=(h, w)) < 0.5
    d[noisy] = np.exp(rng.uniform(np.log(2e-4), np.log(0.05), np.sum(noisy))).astype(np.float32)
    sky = rng.uniform(size=(h, w)) < 0.12
    d[sky] = 0.0
    if hostile:   # +Inf beside sky: its weight is 0 and Inf * 0 is NaN
        ys, xs = np.nonzero(np.isinf(img[..., :3].astype(np.float32)).any(-1))
        for y, x in zip(ys[::2], xs[::2]):
            d[max(y - 1, 0):y + 2, max(x - 1, 0):x + 2] = 0.0
            d[y, x] = 0.004
            img[y, x, 3] = np.float16(2.0)
    yy, xx = np.mgrid[0:h, 0:w] / np.array([max(h - 1, 1), max(w - 1, 1)])[:, None, None]
    n = np.stack([np.sin(3 * xx) * 0.6, np.cos(2 * yy) * 0.5, np.ones_like(xx)], -1)
    n /= np.linalg.norm(n, axis=-1, keepdims=True)
    np_ = rng.uniform(size=(h, w))
    n[np_ < 0.08] *= -1.0                                           # flipped: dp = 0
    n[(np_ >= 0.08) & (np_ < 0.1)] = rng.uniform(-2e-3, 2e-3, (np.sum((np_ >= 0.08) & (np_ < 0.1)), 3))   # near the zero vector
    n += rng.normal(0, 0.02, n.shape) * (np_ >= 0.1)[..., None]
    q = np.clip(np.round((n * 0.5 + 0.5) * 1023.0), 0, 1023).astype(np.uint32)
    gn = ((rng.integers(0, 4, (h, w)).astype(np.uint32) << 30) | (q[..., 0] << 20) | (q[..., 1] << 10) | q[..., 2])[..., None]

    view, jitter = view_constants(w, h, frame_index, (0.1, 1.0 + 0.01 * frame_index, 5.0), (0.1, 1.0 + 0.01 * (frame_index - 1), 5.03))
    fc = frame_constants(sample_offset_pixels=jitter, frame_index=frame_index, view=view)
    inputs = {"input_tex": (img, F16), "depth_tex": (d[..., None], DEPTH), "geometric_normal_tex": (gn, A2R10G10B10)}
    outputs = {"output_tex": (w, h, R11G11B10)}
    offs = offsets()

    def reference(rows=None):
        return ref.spatial_cleanup(img.astype(np.float64), d[..., None].astype(np.float64), gn, offs, view["view_to_clip"][1, 1],
                                   view["clip_to_view"][3, 2], frame_index, rows=rows)
    return inputs, outputs, fc, {"spatial_resolve_offsets": offs}, reference


# ---------------------------------------------------------------- comparison
def compare(got_words, value, slack, mask, what):
    """got R11G11B10 words (H, W, 1) against the float64 reference: per channel, the stored code lies between the product codes of
    value - slack and value + slack (NaN: the product stores 0).  Returns the number of texel-channels compared."""
    got = ref.r11g11b10_codes(got_words[..., 0])
    keep = ~mask
    n = 0
    for ch, m in enumerate(MBITS):
        v, s, g = value[..., ch], slack[..., ch], got[..., ch]
        lo, hi = product_codes(np.where(np.isnan(v), np.nan, v - s), m), product_codes(v + s, m)
        nan = np.isnan(v)
        lo, hi = np.where(nan, 0, lo), np.where(nan, 0, hi)
        bad = keep & ((g < lo) | (g > hi))
        if bad.any():
            i = tuple(np.argwhere(bad)[0])
            raise AssertionError(f"{what} channel {ch}: {int(bad.sum())} of {int(keep.sum())} texels off; first at (y, x) = {i}: got code "
                                 f"{int(g[i])} ({ref.uf_decode(g[i], m)!r}), want codes {int(lo[i])}..{int(hi[i])} for {v[i]!r} +- {s[i]:.3g}")
        n += int(keep.sum())
    return n


def check_mask(mask, what, limit=0.01):
    frac = float(mask.mean()) if mask.size else 0.0
    assert frac <= limit, f"{what}: {mask.sum()} of {mask.size} texels near a decision ({100 * frac:.2f} %)"
    return int(mask.sum())


CPU_CASES = [(1, 37, 23, 0), (2, 64, 40, 1), (3, 40, 24, 2), (4, 61, 37, 3), (5, 32, 21, 6), (6, 48, 33, 7, False)]


def case_id(c):
    return "-".join(str(a) for a in c[1:])


def check_case(runner_, args, bands=None):
    inputs, outputs, fc, ptrs, reference = built = case_cleanup(*args)
    got = runner_.run("cleanup", inputs, outputs, (), fc, pointers=ptrs)
    masked, n, stats = 0, 0, []
    for y0, y1 in bands or [(None, None)]:
        outs, mask, st = reference(rows=None if y0 is None else (y0, y1))
        masked += check_mask(mask, "cleanup")
        n += compare(got["output_tex"][y0:y1], *outs["output_tex"], mask, f"{runner_.lib.backend} cleanup rows {y0}:{y1}")
        stats.append(st)
    assert n > 0
    return got, masked, built, stats


def test_cases_reach_every_path():
    """The synthetic cases reach: the pass-through on `w >= 8` and on sky; both kernel scales; every `filter_idx`; every sample count
    2..8 that `w < 8` allows (4..8); every quad index with several frame indices; flipped normals whose weight is 0; and the NaN of
    Inf * 0 in the weighted sum (which the product stores as 0, DESIGN §8).  A weight sum of 0 is never reached: see
    `test_cleanup_weight_sum_is_never_zero`."""
    through = fidx = sc = nan = ks2 = ks1 = 0
    fidx_seen, sc_seen = set(), set()
    for a in CPU_CASES:
        outs, mask, st = case_cleanup(*a)[4]()
        through += int(st["through"].sum())
        nan += int(st["filtered_nan"].sum())
        assert not st["wsum_zero"].any()
        filt = ~st["through"]
        ks2 += int((filt & (st["kernel_scale"] == 2)).sum()); ks1 += int((filt & (st["kernel_scale"] == 1)).sum())
        sc_seen |= set(st["sample_count"][filt].tolist())
        fidx_seen |= set(st["filter_idx"][filt].tolist())
    assert fidx_seen == set(range(8)), fidx_seen
    assert sc_seen == {4, 5, 6, 7, 8}, sc_seen
    assert through >= 200 and ks2 >= 200 and ks1 >= 200, (through, ks1, ks2)
    assert nan >= 4, nan


def test_cleanup_weight_sum_is_never_zero():
    """spatial_cleanup.hlsl:48 reads offset (0, 0) first for every quad index and filter_idx, so the centre is always sample 0, with
    depth weight exp2(0) = 1 and `dp = saturate(dot(n, n))`; no A2R10G10B10 code decodes to a vector whose float32 `dot(n, n)^3` is 0,
    so `wsum > 0` and `vsum / wsum` is NaN only when a tap is Inf or NaN."""
    offs = offsets()
    for f in range(8):
        for q in range(4):
            assert list(offs[q * 16 + 64 * f, :2]) == [0, 0], (f, q)
    c = (np.arange(1024, dtype=np.float32) / np.float32(1023.0)) * np.float32(2.0) - np.float32(1.0)
    smallest = np.min(np.abs(c))
    dp = np.float32(3.0) * smallest * smallest
    assert dp * dp * dp > 0, smallest


@pytest.mark.parametrize("case", CPU_CASES, ids=case_id)
def test_cleanup_matches_reference_cpu(cpu_runners, case):
    masked = [check_case(r, case)[1] for r in cpu_runners]
    assert masked[0] == masked[1] and masked[0] <= 8, masked


# ---------------------------------------------------------------- the encoder, exhaustively, through R6's pass-through
def encoder_inputs():
    k = np.arange(65536, dtype=np.uint32)
    rgba = np.stack([k, (k + 21845) % 65536, (k + 43690) % 65536, np.full_like(k, 0x4800)], -1).astype(np.uint16)   # alpha 8.0
    img = rgba.reshape(256, 256, 4).view(np.float16)
    inputs = {"input_tex": (img, F16), "depth_tex": (np.full((256, 256, 1), 0.5, np.float32), DEPTH),
              "geometric_normal_tex": (np.zeros((256, 256, 1), np.uint32), A2R10G10B10)}
    return img, inputs


def check_encoder(runner_):
    img, inputs = encoder_inputs()
    got = runner_.run("cleanup", inputs, {"output_tex": (256, 256, R11G11B10)}, (), frame_constants(), pointers={"spatial_resolve_offsets": offsets()})
    codes = ref.r11g11b10_codes(got["output_tex"][..., 0])
    for ch, m in enumerate(MBITS):
        v = img[..., ch].astype(np.float64)
        spec = ref.uf_encode_trunc(v, m)
        g = codes[..., ch]
        differ = g != spec
        # the documented departure and nothing else: every NaN (2 x 1023 f16 codes) stores as 0, +Inf as the largest finite value
        assert np.array_equal(differ, np.isnan(v) | (v == np.inf)), f"{runner_.lib.backend} channel {ch}: {np.argwhere(differ & ~np.isnan(v) & (v != np.inf))[:5].tolist()}"
        assert int(np.isnan(v).sum()) == 2046 and np.all(g[np.isnan(v)] == 0)
        assert np.all(g[v == np.inf] == (30 << m) | ((1 << m) - 1))
        # every finite non-negative value decodes to itself truncated: at most one mantissa ulp below, never above
        fin = np.isfinite(v) & (v >= 0)
        dv = ref.uf_decode(g[fin], m)
        assert np.all(dv <= v[fin]) and np.all((v[fin] - dv) <= np.maximum(np.ldexp(1.0, -14 - m), dv * 2.0 ** -m))


def test_encoder_reference_matches_the_specification():
    """`uf_encode_trunc` against the specification's table, independent of the product: the largest finite values, the smallest
    denormal, the first normal, rounding towards zero, and the special values."""
    for m, top in ((6, 65024.0), (5, 64512.0)):
        assert ref.uf_decode((30 << m) | ((1 << m) - 1), m) == top
        assert ref.uf_encode_trunc(top, m) == (30 << m) | ((1 << m) - 1)
        assert ref.uf_encode_trunc(1e30, m) == (30 << m) | ((1 << m) - 1)
        assert ref.uf_encode_trunc(np.inf, m) == 31 << m and np.isinf(ref.uf_decode(31 << m, m))
        assert ref.uf_encode_trunc(np.nan, m) >> m == 31 and np.isnan(ref.uf_decode(ref.uf_encode_trunc(np.nan, m), m))
        assert ref.uf_encode_trunc(-np.inf, m) == 0 and ref.uf_encode_trunc(-1.0, m) == 0 and ref.uf_encode_trunc(-0.0, m) == 0
        assert ref.uf_decode(1, m) == 2.0 ** (-14 - m) and ref.uf_encode_trunc(2.0 ** (-14 - m) * 0.999, m) == 0
        assert ref.uf_decode(1 << m, m) == 2.0 ** -14 and ref.uf_encode_trunc(2.0 ** -14, m) == 1 << m
        assert ref.uf_encode_trunc(np.nextafter(2.0 ** -14, 0), m) == (1 << m) - 1
        assert ref.uf_encode_trunc(1.0 + 2.0 ** -m * 0.999, m) == 15 << m
        codes = np.arange(31 << m)
        assert np.array_equal(ref.uf_encode_trunc(ref.uf_decode(codes, m), m), codes)


def test_encoder_exhaustive_cpu(cpu_runners):
    for r in cpu_runners:
        check_encoder(r)


# ---------------------------------------------------------------- row bands
BAND_CASES = [((40, 37, 23, 1), [(0, 7), (5, 16), (22, 23)]), ((41, 64, 40, 2), [(3, 10), (17, 40)])]


def check_bands(runner_, args, bands):
    inputs, outputs, fc, ptrs, _ = case_cleanup(*args)
    full = runner_.run("cleanup", inputs, outputs, (), fc, pointers=ptrs)["output_tex"]
    for y0, y1 in bands:
        part = runner_.run("cleanup", inputs, outputs, (), fc, scissor=(y0, y1), sentinel=0x5A, pointers=ptrs)["output_tex"]
        a, s = full.view(np.uint8).reshape(full.shape[0], -1), part.view(np.uint8).reshape(full.shape[0], -1)
        assert np.array_equal(a[y0:y1], s[y0:y1]), f"{runner_.lib.backend} rows [{y0}, {y1}) differ from the full run"
        assert np.all(s[:y0] == 0x5A) and np.all(s[y1:] == 0x5A), f"{runner_.lib.backend} wrote outside rows [{y0}, {y1})"


@pytest.mark.parametrize("case", BAND_CASES, ids=lambda c: case_id((None,) + c[0][1:]))
def test_row_bands_cpu(cpu_runners, case):
    for r in cpu_runners:
        check_bands(r, *case)


def test_reference_row_bands_agree():
    *_, reference = case_cleanup(42, 37, 23, 3)
    full, fmask, _ = reference()
    for y0, y1 in ((0, 5), (6, 7), (17, 23)):
        part, pmask, _ = reference(rows=(y0, y1))
        assert np.array_equal(pmask, fmask[y0:y1])
        for i in range(2):
            assert np.array_equal(part["output_tex"][i], full["output_tex"][i][y0:y1], equal_nan=True)


# ---------------------------------------------------------------- the realistic leg: what a rendered frame's cleanup read
REAL_W, REAL_H, REAL_FRAMES = 64, 40, 4


def check_realistic(r):
    """4 frames of the glossy Cornell box with a rising camera; R6 rerun alone on the last frame's inputs reproduces the frame's
    `rtr.resolved` bit for bit and matches the reference."""
    import parity
    from kajiya_b200 import scenes
    scene, view = scenes.cornell_box()
    w = parity.make_world(r.lib, parity.glossy(scene), REAL_W, REAL_H, enable_rtr=True)
    try:
        w.set_blue_noise(scenes.blue_noise()); w.set_spatial_resolve_offsets(offsets())
        for f in range(REAL_FRAMES):
            pos = (0.0, 1.0 + 0.002 * f, 5.0)
            w.render_frame(**dict(view, camera_position=pos))
        cur = f"{(REAL_FRAMES - 1) % 2}"
        im = {n: w.image(n).copy() for n in ("rtr.temporal:" + cur, "depth", "geometric_normal", "rtr.resolved")}
    finally:
        w.close()
    f = REAL_FRAMES - 1
    vc, jitter = view_constants(REAL_W, REAL_H, f, (0.0, 1.0 + 0.002 * f, 5.0), (0.0, 1.0 + 0.002 * (f - 1), 5.0), view["camera_rotation"])
    fc = frame_constants(sample_offset_pixels=jitter, frame_index=f, view=vc)
    inp, dep, gn = im["rtr.temporal:" + cur], im["depth"].reshape(REAL_H, REAL_W, 1), im["geometric_normal"].reshape(REAL_H, REAL_W, 1)
    got = r.run("cleanup", {"input_tex": (inp, F16), "depth_tex": (dep, DEPTH), "geometric_normal_tex": (gn, A2R10G10B10)},
                {"output_tex": (REAL_W, REAL_H, R11G11B10)}, (), fc, pointers={"spatial_resolve_offsets": offsets()})["output_tex"]
    assert np.array_equal(got.reshape(-1), im["rtr.resolved"].reshape(-1).view(np.uint32)), f"{r.lib.backend}: the rerun differs from the frame's rtr.resolved"
    outs, mask, st = ref.spatial_cleanup(inp.astype(np.float64), dep.astype(np.float64), gn, offsets(), vc["view_to_clip"][1, 1], vc["clip_to_view"][3, 2], f)
    check_mask(mask, "realistic cleanup")
    assert (~st["through"]).sum() > 100    # the frame filters most pixels: its history is short
    compare(got, *outs["output_tex"], mask, f"{r.lib.backend} realistic cleanup")


def test_realistic_frame_cpu(cpu_runners):
    for r in cpu_runners:
        check_realistic(r)


# ---------------------------------------------------------------- H100
GPU_LARGE = [(60, 1920, 1080, 5), (61, 1917, 1079, 9)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CPU_CASES + GPU_LARGE, ids=case_id)
def test_cleanup_matches_reference_gpu(gpu_runner, runners, oracle_lib, case):
    """The H100 against the float64 reference (at the large extents on three row bands) and bit for bit against the oracle."""
    bands = None
    if case in GPU_LARGE:
        h = case[2]
        bands = [(0, 12), (h // 2 - 5, h // 2 + 7), (h - 12, h)]
    got, _, (inputs, outputs, fc, ptrs, _), _ = check_case(gpu_runner, case, bands=bands)
    want = runners(oracle_lib).run("cleanup", inputs, outputs, (), fc, pointers=ptrs)
    diff = np.argwhere(got["output_tex"] != want["output_tex"])
    assert not len(diff), (f"{case_id(case)}: GPU differs from the oracle in {len(diff)} words, first at {diff[0].tolist()}: "
                           f"{hex(int(got['output_tex'][tuple(diff[0])]))} against {hex(int(want['output_tex'][tuple(diff[0])]))}")


@pytest.mark.gpu
def test_encoder_exhaustive_gpu(gpu_runner):
    check_encoder(gpu_runner)


@pytest.mark.gpu
@pytest.mark.parametrize("case", BAND_CASES, ids=lambda c: case_id((None,) + c[0][1:]))
def test_row_bands_gpu(gpu_runner, case):
    check_bands(gpu_runner, *case)


@pytest.mark.gpu
def test_realistic_frame_gpu(gpu_runner):
    check_realistic(gpu_runner)
