"""Each TAA pass (T1-T7, "reproject taa" .. "taa") against `taa_reference.py`, a float64 restatement of kajiya's shaders that
shares nothing with the kernels or the oracle.

The passes are driven one at a time through the C-ABI (kjb_create, kjb_image_alloc/upload, kjb_set_frame_constants, the pass,
kjb_image_download) on the oracle and the emulator, and on the H100.  Every output texel and channel must lie within
2 f16 ulps of the reference plus 2^-11 of the largest absolute tap contribution to it; NaN must match NaN.  Texels the reference
marks as near a decision are excluded, counted, and must stay under 1 %.  The inputs are seeded synthetic images that reach what
whole frames do not: pre_exposure_delta != 1, jitter at the pixel corners, off-screen reprojection, exact depth ties and sky,
f16 subnormals, 6e4, negative channels and neighbourhoods whose luma is all negative (where the shader yields NaN).

Also: a scissored run equals the unscissored run on its rows and leaves the other rows alone, and the H100 equals the oracle
bit for bit on every synthetic case.
"""
import numpy as np
import pytest

import taa_reference as ref
from pass_harness import F16, SNORM, DEPTH, RG16, R16, Runners, extent4, frame_constants
from parity import glossy


# ---------------------------------------------------------------- the passes, in the shape the C-ABI harness drives them
PASSES = {   # entry point, image bindings in kjb.h order, float4 constants
    "reproject": ("kjb_pass_taa_reproject", ["history_tex", "reprojection_tex", "depth_tex", "output_tex", "closest_velocity_output"], 2),
    "filter_input": ("kjb_pass_taa_filter_input", ["input_tex", "depth_tex", "output_tex", "dev_output_tex"], 0),
    "filter_history": ("kjb_pass_taa_filter_history", ["input_tex", "output_tex"], 2),
    "input_prob": ("kjb_pass_taa_input_prob", ["input_tex", "filtered_input_tex", "filtered_input_dev_tex", "history_tex",
                                               "filtered_history_tex", "reprojection_tex", "depth_tex", "smooth_var_history_tex",
                                               "velocity_history_tex", "output_tex"], 1),
    "prob_filter": ("kjb_pass_taa_prob_filter", ["input_tex", "output_tex"], 0),
    "prob_filter2": ("kjb_pass_taa_prob_filter2", ["input_tex", "output_tex"], 0),
    "taa": ("kjb_pass_taa", ["input_tex", "history_tex", "reprojection_tex", "closest_velocity_tex", "velocity_history_tex", "depth_tex",
                             "smooth_var_history_tex", "input_prob_tex", "temporal_output_tex", "output_tex", "smooth_var_output_tex",
                             "velocity_output_tex"], 2),
}
OUTPUTS = {"reproject": ("output_tex", "closest_velocity_output"), "filter_input": ("output_tex", "dev_output_tex"),
           "filter_history": ("output_tex",), "input_prob": ("output_tex",), "prob_filter": ("output_tex",),
           "prob_filter2": ("output_tex",), "taa": ("temporal_output_tex", "output_tex", "smooth_var_output_tex", "velocity_output_tex")}


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


# ---------------------------------------------------------------- seeded synthetic inputs
def colour(rng, w, h, hostile=True):
    """RGBA16F: smooth gradients, step edges and per-texel noise; with `hostile`, also exact zeros, f16 subnormals, 6e4,
    negative channels, greys (so Cb/Cr cancel) and 4x4 patches whose every texel has negative luma."""
    y, x = np.mgrid[0:h, 0:w] / np.array([max(h - 1, 1), max(w - 1, 1)])[:, None, None]
    c = np.stack([0.2 + 0.8 * x, 0.3 + 0.5 * y, 0.5 + 0.4 * x * y, 0.6 + 0.4 * y], -1)
    c *= np.where(((x * 7).astype(int) + (y * 5).astype(int)) % 2 == 0, 1.0, 3.5)[..., None]       # step edges
    c *= np.exp(rng.normal(0, 0.25, (h, w, 4)))                                                   # noise
    c[..., 3] = rng.uniform(0.0, 1.3, (h, w))
    if hostile:
        pick = rng.uniform(size=(h, w))
        c[pick < 0.04] = 0.0
        c[(pick >= 0.04) & (pick < 0.07), :3] = rng.choice([6e-8, 3e-6, 5.9e-5], size=(np.sum((pick >= 0.04) & (pick < 0.07)), 3))
        c[(pick >= 0.07) & (pick < 0.09), :3] = rng.uniform(3e4, 6e4, (np.sum((pick >= 0.07) & (pick < 0.09)), 3))
        c[(pick >= 0.09) & (pick < 0.14), rng.integers(0, 3)] *= -1.0
        grey = (pick >= 0.14) & (pick < 0.24)
        c[grey, :3] = c[grey, :1]
        for _ in range(max(1, w * h // 600)):                                                      # all-negative luma patches
            px, py = rng.integers(0, max(w - 4, 1)), rng.integers(0, max(h - 4, 1))
            c[py:py + 4, px:px + 4, :3] = np.array([0.05, -0.4, 0.05]) * rng.uniform(0.5, 2.0)
    return c.astype(np.float16)


def reprojection(rng, w, h):
    """RGBA16 SNORM: a uniform uv motion with a gentle gradient (too small to trigger dilation) broken by single-texel spikes,
    so that one lane's diagonal test sees a spike that its neighbour's misses and the wave exchange decides; some vectors point
    off-screen; z is the validity the TAA blend reads."""
    y, x = np.mgrid[0:h, 0:w] / np.array([h, w])[:, None, None]
    v = np.zeros((h, w, 4))
    v[..., 0] = 0.5 / w + 0.02 / w * x
    v[..., 1] = -0.3 / h + 0.02 / h * y
    spike = rng.uniform(size=(h, w)) < 0.04
    v[spike, 0] += rng.choice([-1, 1], np.sum(spike)) * rng.uniform(2.0 / w, 0.2, np.sum(spike))
    v[spike, 1] += rng.uniform(-3.0 / h, 3.0 / h, np.sum(spike))
    off = rng.uniform(size=(h, w)) < 0.02
    v[off, :2] = rng.choice([-0.9, 0.9], (np.sum(off), 2))
    v[..., 2] = rng.uniform(0, 1, (h, w))
    v[..., 3] = rng.uniform(-1, 1, (h, w))
    return np.clip(np.round(v * 32767), -32767, 32767).astype(np.int16)


def depth(rng, w, h):
    """R32F reverse-Z: a few exact levels (ties in every 3x3), noise, and sky (0)."""
    d = rng.choice(np.float32([0.25, 0.5, 0.125, 0.75]), (h, w)).astype(np.float32)
    noisy = rng.uniform(size=(h, w)) < 0.5
    d[noisy] = rng.uniform(0.01, 1.0, np.sum(noisy)).astype(np.float32)
    d[rng.uniform(size=(h, w)) < 0.1] = 0.0
    return d[..., None]


def velocity(rng, w, h, scale=1.0):
    return (rng.normal(0, 3.0 / w, (h, w, 2)) * scale).astype(np.float16)


def positive(rng, w, h, c, lo=1e-4, hi=0.5):
    return np.exp(rng.uniform(np.log(lo), np.log(hi), (h, w, c))).astype(np.float16)


def dec(arr, fmt):
    return ref.decode_snorm16(arr) if fmt == SNORM else arr.astype(np.float64)


# ---------------------------------------------------------------- comparison
def f16_ulp(x):
    a = np.abs(np.asarray(x, np.float64))
    e = np.floor(np.log2(np.maximum(a, 2.0 ** -14)))
    return 2.0 ** (e - 10)


def compare(got_raw, value, scale, mask, what):
    """got (H, W, C raw f16) against the float64 reference; masked texels excluded.  Returns the number compared."""
    C_ = min(got_raw.shape[-1], value.shape[-1])
    got = got_raw[..., :C_].astype(np.float64)
    value, scale = value[..., :C_], scale[..., :C_]
    keep = ~mask[..., None] & np.ones_like(got, bool)
    want16 = value.astype(np.float16).astype(np.float64)
    nan_ref, nan_got = np.isnan(value), np.isnan(got)
    bad_nan = keep & (nan_ref != nan_got)
    assert not bad_nan.any(), f"{what}: NaN mismatch at {np.argwhere(bad_nan)[:5].tolist()} (reference NaN there: {nan_ref[bad_nan][:5]})"
    inf = keep & np.isinf(want16) & ~nan_ref
    assert np.all(got[inf] == want16[inf]), f"{what}: overflow to inf mismatch"
    fin = keep & ~nan_ref & ~np.isinf(want16)
    tol = 2.0 * f16_ulp(value) + 2.0 ** -11 * scale
    err = np.where(fin, np.abs(got - value), 0.0)
    bad = err > tol
    if bad.any():
        i = tuple(np.argwhere(bad)[0])
        worst = tuple(np.unravel_index(np.argmax(err / tol), err.shape))
        raise AssertionError(f"{what}: {int(bad.sum())} of {int(fin.sum())} texel-channels off; first at (y, x, c) = {i}: got "
                             f"{got[i]!r}, want {value[i]!r} +- {tol[i]:.3g}; worst {worst}: got {got[worst]!r}, want {value[worst]!r} "
                             f"+- {tol[worst]:.3g}")
    return int(fin.sum())


def check_mask(mask, what, limit=0.01):
    frac = float(mask.mean()) if mask.size else 0.0
    assert frac <= limit, f"{what}: {mask.sum()} of {mask.size} texels near a decision ({100 * frac:.2f} %)"
    return int(mask.sum())


# ---------------------------------------------------------------- cases: one builder per pass -> (inputs, outputs, consts, fc, reference)
def case_reproject(seed, iw, ih, ow, oh, ped=1.0):
    rng = np.random.default_rng(seed)
    hist = colour(rng, ow, oh)
    hist[..., 3] = rng.uniform(-0.2, 1.5, (oh, ow))
    rep, dep = reprojection(rng, iw, ih), depth(rng, iw, ih)
    its, ots = extent4(iw, ih), extent4(ow, oh)
    inputs = {"history_tex": (hist, F16), "reprojection_tex": (rep, SNORM), "depth_tex": (dep, DEPTH)}
    outputs = {"output_tex": (ow, oh, F16), "closest_velocity_output": (ow, oh, RG16)}
    fc = frame_constants(pre_exposure_delta=ped)

    def reference(rows=None):
        return ref.reproject_history(dec(hist, F16), dec(rep, SNORM), dec(dep, DEPTH), its, ots, ped, rows=rows)
    return inputs, outputs, (its, ots), fc, reference


def case_filter_input(seed, w, h):
    rng = np.random.default_rng(seed)
    inp, dep = colour(rng, w, h), depth(rng, w, h)
    inputs = {"input_tex": (inp, F16), "depth_tex": (dep, DEPTH)}
    outputs = {"output_tex": (w, h, F16), "dev_output_tex": (w, h, F16)}

    def reference(rows=None):
        return ref.filter_input(dec(inp, F16), dec(dep, DEPTH), rows=rows)
    return inputs, outputs, (), None, reference


def case_filter_history(seed, iw, ih, ow, oh):
    """history extent (ow, oh) -> filtered at the TAA input extent (iw, ih)"""
    rng = np.random.default_rng(seed)
    hist = colour(rng, ow, oh)
    its, ots = extent4(ow, oh), extent4(iw, ih)
    inputs = {"input_tex": (hist, F16)}
    outputs = {"output_tex": (iw, ih, F16)}

    def reference(rows=None):
        return ref.filter_history(dec(hist, F16), its, ots, rows=rows)
    return inputs, outputs, (its, ots), None, reference


def case_input_prob(seed, iw, ih, ow, oh, jitter, dt):
    rng = np.random.default_rng(seed)
    fin, fdev = colour(rng, iw, ih, hostile=False), positive(rng, iw, ih, 4, 1e-3, 0.3)
    fhist = (fin.astype(np.float32) * np.exp(rng.normal(0, 0.05, fin.shape))).astype(np.float16)
    rep = reprojection(rng, iw, ih)
    svar, vel = positive(rng, ow, oh, 4, 1e-5, 0.1), velocity(rng, ow, oh, 60.0)
    its = extent4(iw, ih)
    inputs = {"input_tex": (colour(rng, iw, ih), F16), "filtered_input_tex": (fin, F16), "filtered_input_dev_tex": (fdev, F16),
              "history_tex": (colour(rng, ow, oh), F16), "filtered_history_tex": (fhist, F16), "reprojection_tex": (rep, SNORM),
              "depth_tex": (depth(rng, iw, ih), DEPTH), "smooth_var_history_tex": (svar, F16), "velocity_history_tex": (vel, RG16)}
    outputs = {"output_tex": (iw, ih, R16)}
    fc = frame_constants(delta_time_seconds=dt, sample_offset_pixels=jitter)

    def reference(rows=None):
        return ref.input_prob(dec(fin, F16), dec(fdev, F16), dec(fhist, F16), dec(rep, SNORM), dec(svar, F16), dec(vel, RG16),
                              its, jitter, dt, rows=rows)
    return inputs, outputs, (its,), fc, reference


def case_prob_filter(seed, w, h, second):
    rng = np.random.default_rng(seed)
    p = rng.uniform(0, 1, (h, w, 1))
    p[rng.uniform(size=(h, w)) < 0.3] = 0.0
    p[rng.uniform(size=(h, w)) < 0.05] = 1.0
    p = p.astype(np.float16)
    inputs = {"input_tex": (p, R16)}
    outputs = {"output_tex": (w, h, R16)}

    def reference(rows=None):
        return (ref.filter_prob2 if second else ref.filter_prob)(dec(p, R16), rows=rows)
    return inputs, outputs, (), None, reference


def case_taa(seed, iw, ih, ow, oh, jitter, dt):
    rng = np.random.default_rng(seed)
    inp = colour(rng, iw, ih)
    hist = colour(rng, ow, oh, hostile=False)
    hist[..., 3] = rng.choice([0.0, 0.5, 1.0, 3.0, 7.9, -0.5], (oh, ow))
    rep = reprojection(rng, iw, ih)
    cvel = (ref.decode_snorm16(reprojection(rng, ow, oh))[..., :2]).astype(np.float16)
    vhist, svar = velocity(rng, ow, oh, 60.0), positive(rng, ow, oh, 4, 1e-5, 0.2)
    prob = rng.uniform(0, 1, (ih, iw, 1))
    prob[rng.uniform(size=(ih, iw)) < 0.2] = rng.choice([0.0, 0.5, 1.0])
    prob = prob.astype(np.float16)
    its, ots = extent4(iw, ih), extent4(ow, oh)
    inputs = {"input_tex": (inp, F16), "history_tex": (hist, F16), "reprojection_tex": (rep, SNORM), "closest_velocity_tex": (cvel, RG16),
              "velocity_history_tex": (vhist, RG16), "depth_tex": (depth(rng, iw, ih), DEPTH), "smooth_var_history_tex": (svar, F16),
              "input_prob_tex": (prob, R16)}
    outputs = {"temporal_output_tex": (ow, oh, F16), "output_tex": (ow, oh, F16), "smooth_var_output_tex": (ow, oh, F16),
               "velocity_output_tex": (ow, oh, RG16)}
    fc = frame_constants(delta_time_seconds=dt, sample_offset_pixels=jitter)

    def reference(rows=None):
        return ref.taa(dec(inp, F16), dec(hist, F16), dec(rep, SNORM), dec(cvel, RG16), dec(vhist, RG16), dec(svar, F16), dec(prob, R16),
                       its, ots, jitter, dt, rows=rows)
    return inputs, outputs, (its, ots), fc, reference


BUILDERS = {"reproject": case_reproject, "filter_input": case_filter_input, "filter_history": case_filter_history,
            "input_prob": case_input_prob, "prob_filter": lambda s, w, h: case_prob_filter(s, w, h, False),
            "prob_filter2": lambda s, w, h: case_prob_filter(s, w, h, True), "taa": case_taa}

CORNERS = [(0.5, 0.5), (-0.5, 0.5), (0.5, -0.5), (-0.5, -0.5), (0.3127, -0.1871)]

# (pass, builder arguments); the extents are (input w, h) then (output w, h) where the pass has two grids
CPU_CASES = (
    [("reproject", (1, 37, 23, 37, 23, ped)) for ped in (1.0, 0.37, 2.5)]
    + [("reproject", (2, 40, 24, 100, 60, 0.37)), ("reproject", (3, 64, 41, 96, 62, 2.5)), ("reproject", (4, 32, 21, 64, 42, 1.0))]
    + [("filter_input", (5, 37, 23)), ("filter_input", (6, 64, 40))]
    + [("filter_history", (7, 37, 23, 37, 23)), ("filter_history", (8, 64, 41, 96, 62)), ("filter_history", (9, 64, 40, 112, 70)),
       ("filter_history", (10, 32, 21, 64, 42)), ("filter_history", (11, 40, 24, 100, 60))]
    + [("input_prob", (12 + i, 37, 23, 37, 23, j, 1.0 / 30.0)) for i, j in enumerate(CORNERS)]
    + [("input_prob", (20, 40, 24, 100, 60, (0.21, 0.43), 0.021))]
    + [("prob_filter", (21, 37, 23)), ("prob_filter2", (22, 37, 23)), ("prob_filter", (23, 64, 40)), ("prob_filter2", (24, 64, 40))]
    + [("taa", (30 + i, 37, 23, 37, 23, j, 1.0 / 45.0)) for i, j in enumerate(CORNERS[:4])]
    + [("taa", (35, 64, 40, 64, 40, (0.137, -0.402), 0.0123)), ("taa", (36, 64, 41, 96, 62, (-0.5, 0.5), 1.0 / 30.0)),
       ("taa", (37, 32, 21, 64, 42, (0.5, -0.5), 1.0 / 60.0)), ("taa", (38, 40, 24, 100, 60, (0.31, 0.07), 0.05)),
       ("taa", (39, 64, 40, 112, 70, (-0.23, -0.5), 1.0 / 24.0))]
)


def case_id(c):
    return f"{c[0]}-" + "-".join(str(a) for a in c[1][1:])


def check_case(runner_, pass_name, args, bands=None):
    """Run one case and compare it with the reference, on every row or on `bands` [(y0, y1), ...] of the output grid."""
    built = BUILDERS[pass_name](*args)
    inputs, outputs, consts, fc, reference = built
    got = runner_.run(pass_name, inputs, outputs, consts, fc)
    masked, n = 0, 0
    for y0, y1 in bands or [(None, None)]:
        outs, mask = reference(rows=None if y0 is None else (y0, y1))
        masked += check_mask(mask, pass_name)
        n += sum(compare(got[b][y0:y1], *outs[b], mask, f"{runner_.lib.backend} {pass_name} {b} rows {y0}:{y1}") for b in OUTPUTS[pass_name])
    assert n > 0
    return got, masked, built


# ---------------------------------------------------------------- the shapes table: which kernel form each case reaches
def test_cases_reach_every_form():
    """Every kernel form is reached: T7 native and upsampling at 1.5, 2, 2.5 with odd heights; T3 tiled, k = 1 at 1.5 and at
    exactly 1.75, k = 2 at 2 and 2.5; T1 native and upsampled."""
    seen = set()
    for p, a in CPU_CASES:
        if p == "filter_history":
            iw, ih, ow, oh = a[1:5]
            k = ref.filter_history_kernel_radius(extent4(ow, oh), extent4(iw, ih))
            seen.add(("T3", "tiled" if (iw, ih) == (ow, oh) else f"k{k}", ow / iw))
        if p in ("taa", "reproject"):
            iw, ih, ow, oh = a[1:5]
            seen.add(("T7" if p == "taa" else "T1", "native" if (iw, ih) == (ow, oh) else "up", ow / iw, oh % 2 or ih % 2))
    for want in [("T3", "tiled", 1.0), ("T3", "k1", 1.5), ("T3", "k1", 1.75), ("T3", "k2", 2.0), ("T3", "k2", 2.5)]:
        assert want in seen, want
    assert {("T7", "up", r) for r in (1.5, 2.0, 2.5)} <= {s[:3] for s in seen}
    assert any(s[0] == "T7" and s[1] == "native" and s[3] for s in seen) and any(s[0] == "T7" and s[1] == "up" and s[3] for s in seen)
    assert {("T1", "native"), ("T1", "up")} <= {s[:2] for s in seen}
    assert ref.filter_history_kernel_radius(extent4(112, 70), extent4(64, 40)) == 1   # 1.75 is not > 1.75
    # on the H100 also: 16-byte aligned rows (bulk row copies), ragged ones (guarded loads), and the upsampling shapes of the benchmarks
    large = {(p, a[1:5] if p in ("reproject", "taa", "filter_history") else a[1:3]) for p, a in GPU_LARGE}
    for p in ("reproject", "taa", "filter_history"):
        assert {(p, e) for e in [(1920, 1080, 1920, 1080), (1917, 1079, 1917, 1079), (1280, 720, 1920, 1080), (960, 540, 1920, 1080),
                                 (2560, 1440, 3840, 2160)]} <= large, p
    for p in ("filter_input", "input_prob", "prob_filter", "prob_filter2"):
        assert any(q == p and e[:2] == (1920, 1080) for q, e in large) and any(q == p and e[:2] == (1917, 1079) for q, e in large), p


def test_cases_reach_the_shaders_nan():
    """The all-negative-luma neighbourhoods make the shader divide 0 by 0 (filter_input.hlsl:64, filter_history.hlsl:44): some
    filter input and filter history cases must have NaN in their reference, or the NaN comparison (and the canonical f16 NaN of
    kjb_numeric.h it checks on the H100) would test nothing."""
    for p in ("filter_input", "filter_history"):
        nan = 0
        for q, a in CPU_CASES:
            if q == p:
                outs, _ = BUILDERS[q](*a)[4]()
                nan += int(np.isnan(outs["output_tex"][0]).any(-1).sum())
        assert nan >= 4, (p, nan)


@pytest.mark.parametrize("case", CPU_CASES, ids=case_id)
def test_pass_matches_reference_cpu(cpu_runners, case):
    """Oracle and emulator against the float64 reference; the synthetic inputs keep the texels near a decision at 0-2."""
    masked = [check_case(r, *case)[1] for r in cpu_runners]
    assert masked[0] == masked[1] and masked[0] <= 2, masked


# ---------------------------------------------------------------- row bands
BAND_CASES = [("reproject", (40, 64, 41, 96, 62, 0.37), [(0, 13), (5, 30), (6, 9), (37, 62)]),
              ("reproject", (41, 37, 23, 37, 23, 2.5), [(5, 17), (6, 23)]),
              ("filter_input", (42, 37, 23), [(0, 7), (5, 16), (11, 23)]),
              ("filter_history", (43, 40, 24, 100, 60), [(3, 10), (17, 24)]),
              ("filter_history", (44, 64, 40, 112, 70), [(0, 5), (21, 40)]),
              ("input_prob", (45, 37, 23, 37, 23, (0.5, -0.5), 0.02), [(1, 8), (19, 23)]),
              ("prob_filter", (46, 37, 23), [(2, 11), (20, 23)]),
              ("prob_filter2", (47, 37, 23), [(0, 3), (9, 22)]),
              ("taa", (48, 64, 41, 96, 62, (0.5, 0.5), 0.02), [(0, 6), (5, 40), (37, 62)]),
              ("taa", (49, 37, 23, 37, 23, (-0.5, 0.25), 0.02), [(6, 7), (10, 23)])]


def check_bands(runner_, pass_name, args, bands):
    inputs, outputs, consts, fc, _ = BUILDERS[pass_name](*args)
    full = runner_.run(pass_name, inputs, outputs, consts, fc)
    for y0, y1 in bands:
        part = runner_.run(pass_name, inputs, outputs, consts, fc, scissor=(y0, y1), sentinel=0x5A)
        for b in OUTPUTS[pass_name]:
            a, s = full[b].view(np.uint8).reshape(full[b].shape[0], -1), part[b].view(np.uint8).reshape(full[b].shape[0], -1)
            assert np.array_equal(a[y0:y1], s[y0:y1]), f"{runner_.lib.backend} {pass_name} {b}: rows [{y0}, {y1}) differ from the full run"
            assert np.all(s[:y0] == 0x5A) and np.all(s[y1:] == 0x5A), f"{runner_.lib.backend} {pass_name} {b}: wrote outside rows [{y0}, {y1})"


@pytest.mark.parametrize("case", BAND_CASES, ids=lambda c: f"{c[0]}-" + "-".join(str(a) for a in c[1][1:5]))
def test_row_bands_cpu(cpu_runners, case):
    for r in cpu_runners:
        check_bands(r, *case)


# ---------------------------------------------------------------- H100
GPU_LARGE = [("reproject", (60, 1920, 1080, 1920, 1080, 0.37)), ("reproject", (61, 1917, 1079, 1917, 1079, 2.5)),
             ("reproject", (62, 1280, 720, 1920, 1080, 1.0)), ("reproject", (63, 960, 540, 1920, 1080, 0.37)),
             ("reproject", (64, 2560, 1440, 3840, 2160, 2.5)),
             ("filter_input", (65, 1920, 1080)), ("filter_input", (66, 1917, 1079)),
             ("filter_history", (67, 1920, 1080, 1920, 1080)), ("filter_history", (68, 1917, 1079, 1917, 1079)),
             ("filter_history", (69, 1280, 720, 1920, 1080)), ("filter_history", (70, 960, 540, 1920, 1080)),
             ("filter_history", (71, 2560, 1440, 3840, 2160)),
             ("input_prob", (72, 1920, 1080, 1920, 1080, (0.5, -0.5), 0.02)), ("input_prob", (73, 1917, 1079, 1917, 1079, (0.11, 0.37), 0.03)),
             ("prob_filter", (74, 1917, 1079)), ("prob_filter2", (75, 1917, 1079)), ("prob_filter", (76, 1920, 1080)), ("prob_filter2", (77, 1920, 1080)),
             ("taa", (78, 1920, 1080, 1920, 1080, (0.5, 0.5), 0.02)), ("taa", (79, 1917, 1079, 1917, 1079, (-0.5, -0.5), 1.0 / 30.0)),
             ("taa", (80, 1280, 720, 1920, 1080, (0.31, -0.12), 1.0 / 60.0)), ("taa", (81, 960, 540, 1920, 1080, (-0.5, 0.5), 0.011)),
             ("taa", (82, 2560, 1440, 3840, 2160, (0.25, 0.5), 0.02))]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CPU_CASES + GPU_LARGE, ids=case_id)
def test_pass_matches_reference_gpu(gpu_runner, runners, oracle_lib, case):
    """The H100 against the float64 reference (at the large extents on three row bands: top, middle, bottom), and bit for bit
    against the oracle on the same inputs (every row)."""
    bands = None
    if case in GPU_LARGE:
        h = case[1][4] if case[0] in ("reproject", "taa") else case[1][2]
        bands = [(0, 12), (h // 2 - 5, h // 2 + 7), (h - 12, h)]
    got, _, (inputs, outputs, consts, fc, _) = check_case(gpu_runner, *case, bands=bands)
    want = runners(oracle_lib).run(case[0], inputs, outputs, consts, fc)
    for b in OUTPUTS[case[0]]:
        g, w = got[b].view(np.uint16 if got[b].dtype == np.float16 else np.uint8), want[b].view(np.uint16 if want[b].dtype == np.float16 else np.uint8)
        diff = np.argwhere(g != w)
        assert not len(diff), (f"{case_id(case)} {b}: GPU differs from the oracle in {len(diff)} words, first at {diff[0].tolist()}: "
                               f"{hex(int(g[tuple(diff[0])]))} against {hex(int(w[tuple(diff[0])]))}")


@pytest.mark.gpu
@pytest.mark.parametrize("case", BAND_CASES, ids=lambda c: f"{c[0]}-" + "-".join(str(a) for a in c[1][1:5]))
def test_row_bands_gpu(gpu_runner, case):
    check_bands(gpu_runner, *case)


# ---------------------------------------------------------------- the realistic leg: the inputs a rendered frame's TAA read
def _halton_offset(frame_idx):
    """the frame driver's jitter: Halton(2, 3) - 0.5 of (frame_idx % 128) + 1, in float32 (world_renderer.rs:425-428)"""
    def radical_inverse(n, base):
        val, inv_base = np.float32(0), np.float32(1) / np.float32(base)
        inv_bi = inv_base
        while n > 0:
            val = np.float32(val + np.float32(n % base) * inv_bi)
            n = int(np.float32(n) * inv_base)
            inv_bi = np.float32(inv_bi * inv_base)
        return val
    i = frame_idx % 128 + 1
    return (float(np.float32(radical_inverse(i, 2) - np.float32(0.5))), float(np.float32(radical_inverse(i, 3) - np.float32(0.5))))


REAL_W, REAL_H, REAL_OW, REAL_OH, REAL_FRAMES = 64, 40, 96, 60, 4


def realistic_passes(lib):
    """Render 4 frames of the glossy Cornell box with a rising camera and 1.5x temporal upsampling; return, for every TAA pass of
    the last frame, the builder tuple of that pass on the images it read, and the images it wrote."""
    import parity
    from kajiya_b200 import scenes
    scene, view = scenes.cornell_box()
    w = parity.make_world(lib, glossy(scene), REAL_W, REAL_H, enable_taa=True, enable_rtr=True, spatial_reuse_pass_count=2,
                          upscale=(REAL_OW, REAL_OH))
    try:
        for f in range(REAL_FRAMES):
            w.render_frame(**dict(view, camera_position=(0.0, 1.0 + 0.002 * f, 5.0)))
        im = {n: w.image(n).copy() for n in w.image_names() if n.startswith("taa") or n in ("depth", "reprojection_map", "rtdgi.spatial_filtered")}
    finally:
        w.close()
    # ping-pong images: frame f writes "<name>:<f % 2>" and reads "<name>:<(f + 1) % 2>" (renderers/mod.rs:73-103); "taa" reads the
    # twice-filtered probability (taa.rs:127-160 binds the block's result, prob_filtered2, to `input_prob_img`)
    cur, hist = f"{(REAL_FRAMES - 1) % 2}", f"{REAL_FRAMES % 2}"
    fc = frame_constants(sample_offset_pixels=_halton_offset(REAL_FRAMES - 1))
    jitter = tuple(float(v) for v in fc[176:178])
    its, ots = extent4(REAL_W, REAL_H), extent4(REAL_OW, REAL_OH)
    inp, rep, dep = im["rtdgi.spatial_filtered"], im["reprojection_map"], im["depth"]
    o = lambda fmt, big=False: (REAL_OW, REAL_OH, fmt) if big else (REAL_W, REAL_H, fmt)
    d = lambda n: dec(im[n], SNORM if n == "reprojection_map" else F16)
    passes = {
        "reproject": ({"history_tex": (im["taa:" + hist], F16), "reprojection_tex": (rep, SNORM), "depth_tex": (dep, DEPTH)},
                      {"output_tex": o(F16, True), "closest_velocity_output": o(RG16, True)}, (its, ots), fc,
                      lambda: ref.reproject_history(d("taa:" + hist), d("reprojection_map"), dep.astype(np.float64), its, ots, 1.0),
                      {"output_tex": "taa.reprojected_history", "closest_velocity_output": "taa.closest_velocity"}),
        "filter_input": ({"input_tex": (inp, F16), "depth_tex": (dep, DEPTH)}, {"output_tex": o(F16), "dev_output_tex": o(F16)}, (), fc,
                         lambda: ref.filter_input(d("rtdgi.spatial_filtered"), dep.astype(np.float64)),
                         {"output_tex": "taa.filtered_input", "dev_output_tex": "taa.filtered_input_deviation"}),
        "filter_history": ({"input_tex": (im["taa.reprojected_history"], F16)}, {"output_tex": o(F16)}, (ots, its), fc,
                           lambda: ref.filter_history(d("taa.reprojected_history"), ots, its), {"output_tex": "taa.filtered_history"}),
        "input_prob": ({"input_tex": (inp, F16), "filtered_input_tex": (im["taa.filtered_input"], F16),
                        "filtered_input_dev_tex": (im["taa.filtered_input_deviation"], F16), "history_tex": (im["taa.reprojected_history"], F16),
                        "filtered_history_tex": (im["taa.filtered_history"], F16), "reprojection_tex": (rep, SNORM), "depth_tex": (dep, DEPTH),
                        "smooth_var_history_tex": (im["taa.smooth_var:" + hist], F16), "velocity_history_tex": (im["taa.velocity:" + hist], RG16)},
                       {"output_tex": o(R16)}, (its,), fc,
                       lambda: ref.input_prob(d("taa.filtered_input"), d("taa.filtered_input_deviation"), d("taa.filtered_history"),
                                              d("reprojection_map"), d("taa.smooth_var:" + hist), d("taa.velocity:" + hist), its, jitter, 1.0 / 60.0),
                       {"output_tex": "taa.input_prob"}),
        "prob_filter": ({"input_tex": (im["taa.input_prob"], R16)}, {"output_tex": o(R16)}, (), fc,
                        lambda: ref.filter_prob(d("taa.input_prob")), {"output_tex": "taa.prob_filtered1"}),
        "prob_filter2": ({"input_tex": (im["taa.prob_filtered1"], R16)}, {"output_tex": o(R16)}, (), fc,
                         lambda: ref.filter_prob2(d("taa.prob_filtered1")), {"output_tex": "taa.prob_filtered2"}),
        "taa": ({"input_tex": (inp, F16), "history_tex": (im["taa.reprojected_history"], F16), "reprojection_tex": (rep, SNORM),
                 "closest_velocity_tex": (im["taa.closest_velocity"], RG16), "velocity_history_tex": (im["taa.velocity:" + hist], RG16),
                 "depth_tex": (dep, DEPTH), "smooth_var_history_tex": (im["taa.smooth_var:" + hist], F16), "input_prob_tex": (im["taa.prob_filtered2"], R16)},
                {"temporal_output_tex": o(F16, True), "output_tex": o(F16, True), "smooth_var_output_tex": o(F16, True), "velocity_output_tex": o(RG16, True)},
                (its, ots), fc,
                lambda: ref.taa(d("rtdgi.spatial_filtered"), d("taa.reprojected_history"), d("reprojection_map"), d("taa.closest_velocity"),
                                d("taa.velocity:" + hist), d("taa.smooth_var:" + hist), d("taa.prob_filtered2"), its, ots, jitter, 1.0 / 60.0),
                {"temporal_output_tex": "taa:" + cur, "output_tex": "taa.this_frame_out", "smooth_var_output_tex": "taa.smooth_var:" + cur,
                 "velocity_output_tex": "taa.velocity:" + cur}),
    }
    return passes, im


def check_realistic(r):
    lib = r.lib
    passes, im = realistic_passes(lib)
    for name, (inputs, outputs, consts, fc, reference, written) in passes.items():
        got = r.run(name, inputs, outputs, consts, fc)
        for b, img in written.items():   # the standalone run reproduces what the frame wrote: these are the inputs it read
            assert np.array_equal(got[b].view(np.uint8), im[img].view(np.uint8)), f"{lib.backend} {name} {b}: standalone run differs from the frame's {img}"
        outs, mask = reference()
        check_mask(mask, f"realistic {name}")
        for b in OUTPUTS[name]:
            compare(got[b], *outs[b], mask, f"{lib.backend} realistic {name} {b}")


def test_realistic_frame_cpu(cpu_runners):
    for r in cpu_runners:
        check_realistic(r)


@pytest.mark.gpu
def test_realistic_frame_gpu(gpu_runner):
    check_realistic(gpu_runner)


@pytest.mark.parametrize("case", [("reproject", (90, 40, 24, 100, 60, 0.37)), ("filter_input", (91, 37, 23)), ("filter_history", (92, 64, 40, 112, 70)),
                                  ("input_prob", (93, 37, 23, 37, 23, (0.5, 0.5), 0.02)), ("prob_filter", (94, 37, 23)), ("prob_filter2", (95, 37, 23)),
                                  ("taa", (96, 40, 24, 100, 60, (-0.5, 0.5), 0.02))], ids=case_id)
def test_reference_row_bands_agree(case):
    """The reference evaluated on a band of rows (how the large GPU cases are checked) equals its whole-grid evaluation there."""
    *_, reference = BUILDERS[case[0]](*case[1])
    full, fmask = reference()
    for y0, y1 in ((0, 5), (5, 11), (6, 7), (17, 23)):
        part, pmask = reference(rows=(y0, y1))
        assert np.array_equal(pmask, fmask[y0:y1])
        for b in OUTPUTS[case[0]]:
            for i in range(2):
                assert np.array_equal(part[b][i], full[b][i][y0:y1], equal_nan=True), (b, y0, y1)
