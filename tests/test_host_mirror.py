"""Independent checks of the C++ host mirror (kajiya_b200/csrc/host/kjb_world.cpp).

Every lockstep parity test runs the SAME mirror on both sides (oracle, emulator and CUDA build all link kjb_world.cpp), so a wiring
mistake in it — a pass in the wrong place, the wrong ping-pong half bound, a constants tuple in the wrong order, a jitter or cascade
constant off — would be invisible to them.  Here the unmodified mirror is linked against a RECORDER backend (tests/mirror/kjb_recorder.cpp:
computes nothing, logs every entry point with its argument bytes) and what it issues is held against two things it shares no code with:

  1. tests/golden/pass_table.json — the render-graph pass declarations extracted mechanically from kajiya's Rust sources
     (tests/golden/make_pass_table.py; binding index = builder call order, crates/lib/kajiya-rg/src/hl.rs:266,324,354-359): per pass
     the resources bound, in order, and the constants tuple; plus the frame's pass order transcribed from
     crates/lib/kajiya/src/world_render_passes.rs:13-292.
  2. a numpy restatement (this file) of prepare_frame_constants (world_renderer.rs:1001-1108), the camera matrices (camera.rs:71-125),
     the TAA jitter (world_renderer.rs:425-428,979-981,1116-1129) and the ircache cascade constants (ircache.rs:126-166).
"""
import ctypes as C, json, os, re, struct, subprocess, shutil
import numpy as np, pytest
import conftest
from kajiya_b200 import scenes
from kajiya_b200._abi import KjbLib
from kajiya_b200.world import World
from camera_reference import camera, view_block

MIRROR = os.path.join(conftest.ROOT, "tests", "mirror")
BASE = 0x7f0000000000


@pytest.fixture(scope="module")
def rec_lib():
    if not shutil.which("g++"):
        pytest.skip("no host compiler")
    build = os.path.join(MIRROR, "_build"); os.makedirs(build, exist_ok=True)
    hdr = open(os.path.join(conftest.ROOT, "include", "kjb.h")).read()
    passes = re.findall(r"^int\s+(kjb_pass_\w+)\s*\(\s*kjb_context\s*\*\s*ctx\s*,\s*const\s+(\w+)\s*\*\s*a\s*\)\s*;", hdr, re.M)
    assert len(passes) > 50
    inc = "".join(f"REC_PASS({fn}, {ty})\n" for fn, ty in passes)
    inc_path = os.path.join(build, "passes.inc")
    if not os.path.exists(inc_path) or open(inc_path).read() != inc:
        open(inc_path, "w").write(inc)
    so = os.path.join(build, "libkjb_rec.so")
    srcs = [os.path.join(MIRROR, "kjb_recorder.cpp"), os.path.join(conftest.ROOT, "kajiya_b200", "csrc", "host", "kjb_world.cpp")]
    deps = srcs + [inc_path, os.path.join(conftest.ROOT, "include", "kjb.h"), os.path.join(conftest.ROOT, "include", "kjb_world.h")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.run(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-I", os.path.join(conftest.ROOT, "include")] + srcs + ["-o", so], check=True)
    lib = KjbLib(so)
    for n, r, a in (("kjb_rec_count", C.c_uint32, []), ("kjb_rec_name", C.c_char_p, [C.c_uint32]), ("kjb_rec_size", C.c_uint32, [C.c_uint32]),
                    ("kjb_rec_data", C.c_void_p, [C.c_uint32]), ("kjb_rec_clear", None, [])):
        getattr(lib.dll, n).restype = r; getattr(lib.dll, n).argtypes = a
    return lib


def drain(lib):
    out = []
    for i in range(lib.dll.kjb_rec_count()):
        n = lib.dll.kjb_rec_size(i)
        out.append((lib.dll.kjb_rec_name(i).decode(), C.string_at(lib.dll.kjb_rec_data(i), n) if n else b""))
    lib.dll.kjb_rec_clear()
    return out


def resources_of(blob, names_by_ptr):
    """(ordered resource names, bytes after the last resource) of one recorded argument struct"""
    found, end = [], 0
    for off in range(0, len(blob) - 7, 8):
        v = struct.unpack_from("<Q", blob, off)[0]
        if BASE < v < BASE + (1 << 44) and (v - BASE) % (1 << 20) == 0 and v in names_by_ptr:
            name, is_image = names_by_ptr[v]
            found.append(name)
            end = off + (24 if is_image_slot(blob, off) else 16)
    return found, blob[end:]


def is_image_slot(blob, off):
    """kjb_image (ptr, w, h, fmt, layers) vs kjb_buffer (ptr, size): formats are 1..16 and layers 1 or 6"""
    if off + 24 > len(blob):
        return False
    w, h, fmt, layers = struct.unpack_from("<4I", blob, off + 8)
    return 1 <= fmt <= 16 and layers in (1, 6) and 0 < w <= 16384 and 0 < h <= 16384 * 6


# ---------------------------------------------------------------------------------------------------- 1. passes and bindings
# rg pass label -> C-ABI entry point (include/kjb.h: one entry per render-graph pass label)
ENTRY = {
    "reprojection map": "kjb_pass_reprojection_map", "copy depth": "kjb_image_copy",
    "clear ircache pool": "kjb_pass_ircache_clear_pool", "scroll cascades": "kjb_pass_ircache_scroll_cascades", "age ircache entries": "kjb_pass_ircache_age_entries",
    "ircache compact": "kjb_pass_ircache_compact", "ircache reset": "kjb_pass_ircache_reset", "ircache trace access": "kjb_pass_ircache_trace_access",
    "ircache validate": "kjb_pass_ircache_validate", "ircache trace": "kjb_pass_ircache_trace", "ircache sum": "kjb_pass_ircache_sum",
    "rtdgi reproject": "kjb_pass_rtdgi_reproject", "extract ssao/2": "kjb_pass_extract_half_res_ssao", "rtdgi validate": "kjb_pass_rtdgi_validate", "rtdgi trace": "kjb_pass_rtdgi_trace",
    "validity integrate": "kjb_pass_rtdgi_validity_integrate", "restir temporal": "kjb_pass_rtdgi_restir_temporal", "restir spatial": "kjb_pass_rtdgi_restir_spatial",
    "restir check": "kjb_pass_rtdgi_restir_check", "restir resolve": "kjb_pass_rtdgi_restir_resolve", "rtdgi temporal": "kjb_pass_rtdgi_temporal", "rtdgi spatial": "kjb_pass_rtdgi_spatial",
    "reflection trace": "kjb_pass_rtr_trace", "reflection validate": "kjb_pass_rtr_validate", "rtr restir temporal": "kjb_pass_rtr_restir_temporal", "reflection resolve": "kjb_pass_rtr_resolve",
    "reflection temporal": "kjb_pass_rtr_temporal", "reflection cleanup": "kjb_pass_rtr_cleanup",
    "reproject taa": "kjb_pass_taa_reproject", "taa filter input": "kjb_pass_taa_filter_input", "taa filter history": "kjb_pass_taa_filter_history", "taa input prob": "kjb_pass_taa_input_prob",
    "taa prob filter": "kjb_pass_taa_prob_filter", "taa prob filter2": "kjb_pass_taa_prob_filter2", "taa": "kjb_pass_taa",
    "extract view normal/2": "kjb_pass_extract_half_res_view_normal", "extract half depth": "kjb_pass_extract_half_res_depth",
}
IRCACHE_BIND_MUT = ["ircache.meta_buf", "ircache.pool_buf", "ircache.reposition_proposal_buf", "ircache.reposition_proposal_count_buf", "GRID", "ircache.entry_cell_buf",
                    "ircache.spatial_buf", "ircache.irradiance_buf", "ircache.life_buf"]   # IrcacheRenderState::bind_mut, ircache.rs:59-78 (asserted against the source below)


class Names:
    """Rust binding expression -> the mirror's resource name, for frame `f` (0-based)."""

    def __init__(self, f, spatial_passes):
        self.f, self.n = f, spatial_passes
        self.grid_cur = "ircache.grid_meta_buf2" if f % 2 == 1 else "ircache.grid_meta_buf"   # after this frame's scroll + swap (ircache.rs:252-268)
        self.grid_prev = "ircache.grid_meta_buf" if f % 2 == 1 else "ircache.grid_meta_buf2"

    def out(self, n): return f"{n}:{self.f % 2}"          # PingPongTemporalResource (renderers/mod.rs:73-103): output_key = name:0 on the first frame, swapped every frame
    def hist(self, n): return f"{n}:{1 - self.f % 2}"

    def common(self, e):
        m = {"reprojection_map": "reprojection_map", "&gbuffer_depth.depth": "depth", "depth_tex": "depth", "depth": "depth", "&gbuffer_depth.gbuffer": "gbuffer", "gbuffer": "gbuffer",
             "&gbuffer_depth.geometric_normal": "geometric_normal", "&*half_view_normal_tex": "half_view_normal", "&*half_depth_tex": "half_depth", "ssao_tex": "ssao",
             "velocity_img": "velocity", "&prev_depth": "reprojection.prev_depth", "&mut prev_depth": "reprojection.prev_depth", "bind | wrc": None}
        return m.get(e, KeyError)

    def rtdgi(self, label, e, k=0):
        o, h = self.out, self.hist
        spatial_in = o("rtdgi.reservoir") if k == 0 else f"rtdgi.reservoir_output{(k - 1) % 2}"
        last = f"rtdgi.reservoir_output{(self.n - 1) % 2}"
        per = {
            "rtdgi temporal": {"input_color": "rtdgi.irradiance", "rt_history_invalidity_tex": o("rtdgi.invalidity")},
            "rtdgi spatial": {"input_color": "rtdgi.temporal_filtered"},
            "rtdgi reproject": {"&history_tex": h("rtdgi.temporal2")},
            "restir spatial": {"reservoir_input_tex": spatial_in, "&mut reservoir_output_tex0": f"rtdgi.reservoir_output{k % 2}"},
            "restir check": {"reservoir_input_tex": last}, "restir resolve": {"reservoir_input_tex": last, "&radiance_tex": o("rtdgi.radiance")},
        }.get(label, {})
        if e in per:
            return per[e]
        m = {"reprojected_history_tex": "rtdgi.reprojected_history", "&reprojected_history_tex": "rtdgi.reprojected_history", "&mut reprojected_history_tex": "rtdgi.reprojected_history",
             "&variance_history_tex": h("rtdgi.temporal2_var"), "&mut temporal_variance_output_tex": o("rtdgi.temporal2_var"), "&mut temporal_filtered_tex": "rtdgi.temporal_filtered",
             "&mut temporal_output_tex": o("rtdgi.temporal2"), "&mut spatial_filtered_tex": "rtdgi.spatial_filtered", "&mut half_ssao_tex": "rtdgi.half_ssao", "&half_ssao_tex": "rtdgi.half_ssao",
             "&mut reservoir_history_tex": h("rtdgi.reservoir"), "&reservoir_history_tex": h("rtdgi.reservoir"), "&ray_history_tex": h("rtdgi.ray"), "sky_cube": "convolved_sky_cube",
             "&mut radiance_history_tex": h("rtdgi.radiance"), "&radiance_history_tex": h("rtdgi.radiance"), "&ray_orig_history_tex": h("rtdgi.ray_orig"),
             "&mut rt_history_validity_pre_input_tex": "rtdgi.rt_history_validity_pre_input", "&rt_history_validity_pre_input_tex": "rtdgi.rt_history_validity_pre_input",
             "&mut rt_history_validity_input_tex": "rtdgi.rt_history_validity_input", "&rt_history_validity_input_tex": "rtdgi.rt_history_validity_input",
             "&mut candidate_radiance_tex": "rtdgi.candidate_radiance", "&candidate_radiance_tex": "rtdgi.candidate_radiance", "&mut candidate_normal_tex": "rtdgi.candidate_normal",
             "&candidate_normal_tex": "rtdgi.candidate_normal", "&mut candidate_hit_tex": "rtdgi.candidate_hit", "&candidate_hit_tex": "rtdgi.candidate_hit",
             "&invalidity_history_tex": h("rtdgi.invalidity"), "&mut invalidity_output_tex": o("rtdgi.invalidity"), "&invalidity_output_tex": o("rtdgi.invalidity"),
             "&hit_normal_history_tex": h("rtdgi.hit_normal"), "&candidate_history_tex": h("rtdgi.candidate"),
             "&mut radiance_output_tex": o("rtdgi.radiance"), "&mut ray_orig_output_tex": o("rtdgi.ray_orig"), "&mut ray_output_tex": o("rtdgi.ray"), "&mut hit_normal_output_tex": o("rtdgi.hit_normal"),
             "&mut reservoir_output_tex": o("rtdgi.reservoir"), "&mut candidate_output_tex": o("rtdgi.candidate"),
             "&mut temporal_reservoir_packed_tex": "rtdgi.temporal_reservoir_packed", "&temporal_reservoir_packed_tex": "rtdgi.temporal_reservoir_packed",
             "bounced_radiance_input_tex": None, "&mut bounced_radiance_output_tex0": None,   # only with RTDGI_RESTIR_SPATIAL_USE_RAYMARCH_COLOR_BOUNCE (off, rtdgi_restir_settings.hlsl:17): a 1x1 dummy upstream, unbound here
             "&mut irradiance_output_tex": "rtdgi.irradiance"}
        return m.get(e, KeyError)

    def rtr(self, label, e, k=0):
        o, h = self.out, self.hist
        m = {"rtdgi_irradiance": "rtdgi.spatial_filtered", "sky_cube": "sky_cube", "&ranking_tile_buf": None, "&scambling_tile_buf": None, "&sobol_buf": None,   # blue-noise-sampler tables: not supplied (DESIGN §8)
             "&mut refl0_tex": "rtdgi.candidate_radiance", "&refl0_tex": "rtdgi.candidate_radiance", "&mut refl1_tex": "rtdgi.candidate_hit", "&refl1_tex": "rtdgi.candidate_hit",
             "&mut refl2_tex": "rtdgi.candidate_normal", "&refl2_tex": "rtdgi.candidate_normal",   # RtdgiCandidates reused as reflection candidates (rtr.rs:105-109)
             "&mut rng_output_tex": o("rtr.rng"), "&rng_history_tex": h("rtr.rng"), "&mut refl_restir_invalidity_tex": "rtr.restir_invalidity", "&self.refl_restir_invalidity_tex": "rtr.restir_invalidity",
             "&ray_orig_history_tex": h("rtr.ray_orig"), "&ray_history_tex": h("rtr.ray"), "&mut irradiance_history_tex": h("rtr.irradiance"), "&irradiance_history_tex": h("rtr.irradiance"),
             "&mut reservoir_history_tex": h("rtr.reservoir"), "&reservoir_history_tex": h("rtr.reservoir"), "&hit_normal_history_tex": h("rtr.hit_normal"),
             "&mut irradiance_output_tex": o("rtr.irradiance"), "&mut ray_orig_output_tex": o("rtr.ray_orig"), "&ray_orig_output_tex": o("rtr.ray_orig"), "&mut ray_output_tex": o("rtr.ray"),
             "&mut hit_normal_output_tex": o("rtr.hit_normal"), "&mut reservoir_output_tex": o("rtr.reservoir"),
             "&history_tex": h("rtr.temporal"), "&self.history_tex": h("rtr.temporal"), "&ray_len_history_tex": h("rtr.ray_len"), "&irradiance_tex": o("rtr.irradiance"), "&ray_tex": o("rtr.ray"),
             "&temporal_reservoir_tex": o("rtr.reservoir"), "&restir_hit_normal_tex": o("rtr.hit_normal"), "&mut resolved_tex": "rtr.resolved", "&self.resolved_tex": "rtr.resolved",
             "&mut self.resolved_tex": "rtr.resolved", "&mut ray_len_output_tex": o("rtr.ray_len"), "&self.ray_len_tex": o("rtr.ray_len"),
             "&mut self.temporal_output_tex": o("rtr.temporal"), "&self.temporal_output_tex": o("rtr.temporal")}
        return m.get(e, KeyError)

    def taa(self, label, e, k=0):
        o, h = self.out, self.hist
        m = {"&history_tex": h("taa"), "&mut reprojected_history_img": "taa.reprojected_history", "&reprojected_history_img": "taa.reprojected_history",
             "&mut closest_velocity_img": "taa.closest_velocity", "&closest_velocity_img": "taa.closest_velocity", "input_tex": "TAA_INPUT",
             "&mut filtered_input_img": "taa.filtered_input", "&filtered_input_img": "taa.filtered_input", "&mut filtered_input_deviation_img": "taa.filtered_input_deviation",
             "&filtered_input_deviation_img": "taa.filtered_input_deviation", "&mut filtered_history_img": "taa.filtered_history", "&filtered_history_img": "taa.filtered_history",
             "&smooth_var_history_tex": h("taa.smooth_var"), "&velocity_history_tex": h("taa.velocity"), "&mut input_prob_img": "taa.input_prob", "&input_prob_img": "PROB_IN",
             "&mut prob_filtered1_img": "taa.prob_filtered1", "&prob_filtered1_img": "taa.prob_filtered1", "&mut prob_filtered2_img": "taa.prob_filtered2",
             "&mut temporal_output_tex": o("taa"), "&mut this_frame_output_img": "taa.this_frame_out", "&mut smooth_var_output_tex": o("taa.smooth_var"), "&mut temporal_velocity_output_tex": o("taa.velocity")}
        return m.get(e, KeyError)

    def ircache(self, label, e, k=0):
        grid = self.grid_cur
        if label == "scroll cascades":
            return {"&state.ircache_grid_meta_buf": self.grid_prev, "&mut state.ircache_grid_meta_buf2": self.grid_cur}.get(e) or self._irc(e, self.grid_prev)
        return self._irc(e, grid)

    def _irc(self, e, grid):
        e2 = re.sub(r"^&(mut )?(state|self)\.", "", e)
        m = {"ircache_meta_buf": "ircache.meta_buf", "ircache_grid_meta_buf": grid, "ircache_entry_cell_buf": "ircache.entry_cell_buf", "ircache_spatial_buf": "ircache.spatial_buf",
             "ircache_irradiance_buf": "ircache.irradiance_buf", "ircache_aux_buf": "ircache.aux_buf", "ircache_life_buf": "ircache.life_buf", "ircache_pool_buf": "ircache.pool_buf",
             "ircache_entry_indirection_buf": "ircache.entry_indirection_buf", "ircache_reposition_proposal_buf": "ircache.reposition_proposal_buf",
             "ircache_reposition_proposal_count_buf": "ircache.reposition_proposal_count_buf", "&mut entry_occupancy_buf": "ircache.entry_occupancy_buf", "&entry_occupancy_buf": "ircache.entry_occupancy_buf",
             "sky_cube": "convolved_sky_cube"}
        return m.get(e2, KeyError)


def expected_bindings(p, names, k=0, ircache_bound=True):
    fam = {"rtdgi.rs": names.rtdgi, "rtr.rs": names.rtr, "taa.rs": names.taa, "ircache.rs": names.ircache, "reprojection.rs": (lambda label, e, k=0: {"&mut output_tex": "reprojection_map"}.get(e, KeyError)), "half_res.rs": names.rtdgi}[p["file"].split("/")[-1]]
    out = []
    for c in p["calls"]:
        if c["m"] in ("constants", "raw_descriptor_set", "dynamic_storage_buffer"):
            continue
        if c["m"] == "bind":          # wrc: USE_WORLD_RADIANCE_CACHE 0 — nothing is bound
            continue
        if c["m"] == "bind_mut":
            if ircache_bound:   # upstream always has a cache; this ABI lets a host leave the block NULL (lookups then contribute 0)
                out += [names.grid_cur if n == "GRID" else n for n in IRCACHE_BIND_MUT]
            continue
        e = c["arg"].split(", vk::ImageAspectFlags")[0].strip()
        r = names.common(e)
        if r is KeyError:
            r = fam(p["label"], e, k)
        assert r is not KeyError, f'{p["label"]}: no mapping for Rust binding `{e}` ({p["file"]}:{p["line"]})'
        if r is not None:
            out.append(r)
    return out


def frame_sequence(feat, frame, spatial_passes):
    """rg pass labels of one frame in the order of prepare_render_graph_standard (world_render_passes.rs:13-292) and the renderers it calls,
    restricted to the hot path (ssgi / shadows / light_gbuffer / post are exercised by their own lockstep tests)."""
    seq = ["reprojection map", "copy depth"]                                                                    # :84-90, reprojection.rs:6-52
    if feat["ircache"]:
        seq += ["clear ircache pool" if frame == 0 else "scroll cascades", "_ircache dispatch args", "age ircache entries", "_prefix scan", "ircache compact"]   # ircache.prepare :99, ircache.rs:233-351
        seq += ["_ircache dispatch args", "ircache reset", "ircache trace access", "ircache validate", "ircache trace"]                                          # trace_irradiance :113-122, ircache.rs:360-487
    seq += ["rtdgi reproject"]                                                                                  # :129
    if feat["ircache"]:
        seq += ["ircache sum"]                                                                                  # :138-140
    # rtdgi.render :146-160, rtdgi.rs:173-554 (GbufferDepth half-res extracts are memoised: first use inside rtdgi when ssgi is off)
    seq += ["extract ssao/2", "extract half depth", "extract view normal/2", "rtdgi validate", "rtdgi trace", "validity integrate", "restir temporal"] + ["restir spatial"] * spatial_passes + \
           ["restir resolve", "rtdgi temporal", "rtdgi spatial"]
    if feat["rtr"]:
        seq += ["reflection trace", "reflection validate", "rtr restir temporal", "reflection resolve", "reflection temporal", "reflection cleanup"]   # :171-205, rtr.rs:90-399
    if feat["taa"]:
        seq += ["reproject taa", "taa filter input", "taa filter history", "taa input prob", "taa prob filter", "taa prob filter2", "taa"]              # :253-263, taa.rs:41-185
    return seq


def test_ircache_bind_order_matches_the_reference():
    """the mirror binds the irradiance-cache buffers in the order the reference's `bind_mut` does (extracted into the fixture by make_pass_table.py)"""
    order = json.load(open(os.path.join(conftest.ROOT, "tests", "golden", "pass_table.json")))["ircache_bind_mut_order"]
    want = [n.split(".")[1] if n != "GRID" else "grid_meta_buf" for n in IRCACHE_BIND_MUT]
    assert [o.replace("ircache_", "") for o in order] == want, order


@pytest.mark.parametrize("feat", [dict(ircache=True, rtr=True, taa=True), dict(ircache=False, rtr=False, taa=False), dict(ircache=False, rtr=True, taa=True)])
def test_mirror_issues_the_reference_passes_with_the_reference_bindings(rec_lib, feat):
    table = {}
    for p in json.load(open(os.path.join(conftest.ROOT, "tests", "golden", "pass_table.json")))["passes"]:
        if p["label"] and p["terminal"]:
            table.setdefault(p["label"], []).append(p)
    W, H, SP = 1920, 1080, 2
    scene, view = scenes.cornell_box()
    w = World(rec_lib, W, H, spatial_reuse_pass_count=SP, enable_ircache=feat["ircache"], enable_rtr=feat["rtr"], enable_taa=feat["taa"])
    scenes.populate(w, scene)
    drain(rec_lib)
    for f in range(4):
        w.render_frame(**view)
        log = [r for r in drain(rec_lib) if r[0].startswith("kjb_pass_") or r[0] == "kjb_image_copy"]
        ptrs = {}
        for n in w.image_names():
            h = w.image_handle(n); ptrs[h.data] = (n, True)
        skip = {"kjb_pass_raster_gbuffer", "kjb_pass_sky_cube", "kjb_pass_convolve_sky", "kjb_pass_brdf_fg_lut"}   # input producers ahead of the hot path
        log = [r for r in log if r[0] not in skip]
        seq = frame_sequence(feat, f, SP)
        names = Names(f, SP)
        # ---- order: one recorded entry point per expected label, in order ("_prefix scan" is one entry point for the reference's three passes)
        got = [r[0] for r in log]
        want = []
        dispatch_args_seen = 0
        for lab in seq:
            if lab == "_ircache dispatch args":
                want.append("kjb_pass_ircache_prepare_age_dispatch_args" if dispatch_args_seen == 0 else "kjb_pass_ircache_prepare_trace_dispatch_args"); dispatch_args_seen += 1
            elif lab == "_prefix scan":
                want.append("kjb_pass_inclusive_prefix_scan_u32")
            elif lab == "extract half depth":
                want.append("FUSED")     # the mirror issues the three half-res extracts as one fused launch when none ran yet this frame
            elif lab in ("extract ssao/2", "extract view normal/2"):
                continue
            else:
                want.append(ENTRY[lab])
        got_n = ["FUSED" if g == "kjb_pass_extract_half_res_fused" else g for g in got]
        assert got_n == want, (f, [(a, b) for a, b in zip(got_n, want) if a != b][:4], len(got_n), len(want))
        # ---- bindings, pass by pass
        k_spatial = 0
        for (fn, blob), lab in zip(log, [l for l in seq if l not in ("extract ssao/2", "extract view normal/2")]):
            if lab in ("_ircache dispatch args", "_prefix scan", "extract half depth"):
                continue
            cands = table[lab]
            p = cands[0]
            bound, tail = resources_of(blob, ptrs)
            k = 0
            if lab == "restir spatial":
                k = k_spatial; k_spatial += 1
            exp = expected_bindings(p, names, k, feat["ircache"])
            if lab == "copy depth":
                exp = [exp[1], exp[0]]     # kjb_image_copy(dst, src)
            if lab.startswith("taa") or lab == "reproject taa":
                exp = ["rtdgi.spatial_filtered" if e == "TAA_INPUT" else ("taa.prob_filtered2" if (e == "PROB_IN" and lab == "taa") else ("taa.input_prob" if e == "PROB_IN" else e)) for e in exp]
            assert bound == exp, (f, lab, f'{p["file"]}:{p["line"]}', [(a, b) for a, b in zip(bound, exp) if a != b][:4], len(bound), len(exp))
            # ---- constants: every `X.desc().extent_inv_extent_2d()` of the tuple, in order, at the head of the bytes that follow the resources
            cons = [c["arg"] for c in p["calls"] if c["m"] == "constants"]
            if cons:
                items = [i.strip() for i in re.sub(r"^\(|\)$", "", cons[0]).split(",") if i.strip()]
                floats = np.frombuffer(tail[:len(tail) // 4 * 4], np.float32)
                pos = None   # unbound (NULL) resource slots may sit between the last bound resource and the constants: find the first tuple, then walk
                for it in items:
                    m = re.match(r"([\w.]+?)(?:\.desc\(\))?\.extent_inv_extent_2d\(\)", it)
                    if not m:
                        break
                    var = m.group(1)
                    half = var in ("invalidity_output_tex", "reservoir_output_tex0")
                    ew, eh = ((W + 1) // 2, (H + 1) // 2) if half else (W, H)
                    want4 = np.array([ew, eh, np.float32(1.0) / np.float32(ew), np.float32(1.0) / np.float32(eh)], np.float32)
                    if pos is None:
                        hits = [i for i in range(0, len(floats) - 3, 2) if np.array_equal(floats[i:i + 4], want4)]
                        assert hits, (lab, it, want4)
                        pos = hits[0]
                    assert np.array_equal(floats[pos:pos + 4], want4), (lab, it, floats[pos:pos + 4], want4)
                    pos += 4
                if lab == "restir spatial":   # (gbuffer size, output size, spatial_reuse_pass_idx, perform_occlusion_raymarch, occlusion_raymarch_importance_only) rtdgi.rs:459-465
                    u = np.frombuffer(tail[pos * 4:pos * 4 + 12], np.uint32)
                    assert list(u) == [k, 1 if k + 1 == SP else 0, 0], (k, u)
    w.close()


# ---------------------------------------------------------------------------------------------------- 2. per-frame constants
def test_frame_constants_against_a_numpy_restatement(rec_lib):
    W, H = 1280, 720
    scene, _ = scenes.cornell_box()
    w = World(rec_lib, W, H, enable_ircache=True)
    scenes.populate(w, scene)
    drain(rec_lib)
    rot = (0.0, float(np.sin(0.3)), 0.0, float(np.cos(0.3)))
    prev_cam, prev_scroll = None, np.zeros((12, 3), np.int64)
    for f in range(5):
        pos = (0.37 * f - 1.0, 1.0 + 0.011 * f, 7.0 - 0.4 * f)
        sun = (0.3, 0.6, 1.0)
        w.render_frame(camera_position=pos, camera_rotation=rot, sun_direction=sun)
        fc = [b for n, b in drain(rec_lib) if n == "kjb_set_frame_constants"]
        assert len(fc) == 1 and len(fc[0]) == 1216
        fl = np.frombuffer(fc[0], np.float32); ui = np.frombuffer(fc[0], np.uint32); si = np.frombuffer(fc[0], np.int32)
        mats = fl[:11 * 16].reshape(11, 4, 4).transpose(0, 2, 1)      # column-major -> [row, col]
        names = ["view_to_clip", "clip_to_view", "view_to_sample", "sample_to_view", "world_to_view", "view_to_world", "clip_to_prev_clip",
                 "prev_view_to_prev_clip", "prev_clip_to_prev_view", "prev_world_to_prev_view", "prev_view_to_prev_world"]
        got = dict(zip(names, mats))
        cam = camera(pos, rot, W, H)
        prev = prev_cam or cam
        want, off, off_clip = view_block(cam, prev, f, W, H)
        for n in names:   # products of up to four matrices built from cos / sin: equal to a few ulps (libm differences), far tighter than any wiring mistake
            assert np.allclose(got[n], want[n], rtol=2e-6, atol=1e-7), (f, n, got[n], want[n])
        for n in ("world_to_view", "view_to_world"):   # no transcendental involved: exact
            assert np.array_equal(got[n].view(np.uint32), want[n].view(np.uint32)), (f, n)
        o = 11 * 16
        assert np.array_equal(fl[o:o + 2], off) and np.array_equal(fl[o + 2:o + 4], off_clip)
        o += 4
        sl = np.float32(np.sqrt(np.float32(sun[0]) ** 2 + np.float32(sun[1]) ** 2 + np.float32(sun[2]) ** 2))
        assert np.allclose(fl[o:o + 3], np.array(sun, np.float32) / sl, rtol=0, atol=1e-7) and fl[o + 3] == 0
        assert ui[o + 4] == f and fl[o + 5] == np.float32(1.0 / 60.0) and ui[o + 7] == 0          # frame_index, delta_time, no triangle lights
        assert abs(float(fl[o + 6]) - np.cos(0.5 * 0.53 * np.pi / 180.0)) < 1e-7                  # sun_angular_radius_cos (world_renderer.rs:1078)
        assert list(fl[o + 8:o + 12]) == [1, 1, 1, 0] and list(fl[o + 12:o + 16]) == [0, 0, 0, 0]   # sun colour multiplier, sky ambient
        assert list(fl[o + 16:o + 19]) == [1, 1, 1]                                               # pre_exposure, _prev, _delta
        o += 24
        assert np.array_equal(fl[o:o + 3], np.array(pos, np.float32)) and fl[o + 3] == 1.0         # ircache_grid_center (ircache.rs:126-131)
        o += 4
        casc = si[o:o + 12 * 8].reshape(12, 2, 4)
        for c in range(12):   # IrcacheRenderer::update_eye_position (ircache.rs:133-157): cell diameter 0.16 / 8 * 2^cascade, origin = floor(eye / diameter) - 16
            d = np.float32(np.float32(0.16 * 0.125) * np.float32(1 << c))
            origin = np.floor(np.array(pos, np.float32) / d).astype(np.int64) - 16
            assert list(casc[c, 0, :3]) == list(origin), (f, c, casc[c, 0], origin)
            assert list(casc[c, 1, :3]) == list(origin - prev_scroll[c]), (f, c)
            prev_scroll[c] = origin
        prev_cam = cam
    w.close()
