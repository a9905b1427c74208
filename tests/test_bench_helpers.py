"""bench.py pieces that can be checked without a GPU."""
import importlib.util, os
import conftest


def _bench():
    spec = importlib.util.spec_from_file_location("bench_under_test", os.path.join(conftest.ROOT, "bench.py"))
    m = importlib.util.module_from_spec(spec); spec.loader.exec_module(m)
    return m


def test_pass_byte_table_covers_every_label_the_frame_driver_emits():
    b = _bench()
    src = open(os.path.join(conftest.ROOT, "kajiya_b200", "csrc", "host", "kjb_world.cpp")).read()
    import re
    labels = set(re.findall(r'RUN(?:_TOP)?\("([^"]+)"', src)) - {"raster simple", "sky cube", "convolve sky", "brdf fg lut", "reference pt"}
    missing = sorted(l for l in labels if l not in b.PASS_BYTES and not l.startswith("_") and l != "tile border all-gather")
    assert missing == [], missing
    F, Hh = 1920 * 1080, 960 * 540
    for l in labels & set(b.PASS_BYTES):
        assert b.pass_bytes(l, F, Hh) >= 0


def test_summarize_builds_the_roofline_from_per_pass_timings():
    b = _bench()
    F, Hh = 1920 * 1080, 960 * 540
    m = dict(workload="atrium_1080p_full", F=F, Hh=Hh, O=F, K=4, ms_total=8.0, ms_e2e=12.0, rays=4_000_000, rays_e2e=4_000_000, launches=160, h2d=32 * F + 1216, d2h=8 * F, streaming=True,
             per_pass={"reflection resolve": 0.5, "restir spatial": 0.1, "tile border all-gather": 0.9}, calls={"reflection resolve": 4, "restir spatial": 8, "tile border all-gather": 4})
    table = {"atrium_1080p_full": {"reflection resolve": {"dram_bytes": 5.0e7, "warp_inst": 2.0e8, "source": "profiles/x.csv"}}}
    e = b.summarize(m, 1, 6585.1, table)
    r = e["roofline"]
    assert r["kernel"] == "reflection resolve"                       # the exchange wait is not a kernel; spatial runs twice but is still smaller
    assert abs(r["algorithmic_bytes_per_launch"] - (36 * F + 60 * Hh)) < 1 and abs(r["achieved"] - (36 * F + 60 * Hh) / 0.5e-3 / 1e9) < 1e-6
    assert r["traffic"] == 5.0e7 and r["traffic_source"] == "profiles/x.csv" and 0 < r["issue_slots"]["frac"] < 1
    assert abs(e["ms_per_step"] - 2.0) < 1e-12 and abs(e["value"] - 4_000_000 / 8e-3) < 1e-3
    e8 = b.summarize(m, 8, 6585.1, table)                            # N > 1: N x the per-GPU peak, no single-GPU ncu table
    assert abs(e8["roofline"]["peak"] - 8 * 6585.1) < 1e-9 and e8["roofline"]["traffic"] is None and abs(e8["roofline"]["frac"] * 8 - r["frac"]) < 1e-12


def test_both_arms_print_the_same_config_and_every_baseline_configuration_has_a_workload():
    b = _bench()
    import json
    base = json.load(open(os.path.join(conftest.ROOT, "BASELINE.json")))
    assert sorted(b.BASELINE_CONFIG.values()) == list(range(len(base["configs"]))) and set(b.CONFIG_SET) == set(b.BASELINE_CONFIG)
    c = b.config_of(b.HEADLINE)
    assert c == b.config_of(b.HEADLINE) and c["baseline_config"] == 2 and c["resolution"] == [1920, 1080]
    r = b.config_of("ruins_4k_upsampled_full")                       # `--temporal-upsampling 1.5` at 4K renders 2560x1440 (main_loop.rs:222-233)
    assert r["resolution"] == [2560, 1440] and r["output_resolution"] == [3840, 2160]


def test_band_compare():
    b = _bench()
    import numpy as np
    a = (np.random.RandomState(1).rand(64, 32, 4) * 1000).astype(np.uint16)
    t = a.copy(); t[:16] = 0                                         # rank 1 of 4 owns rows 16..32: other bands may differ
    assert b.band_compare(a, t, 64, 1, 4, False)[:2] == (True, True)
    t[20, 3, 0] ^= 1
    ok, exact, *_ = b.band_compare(a, t, 64, 1, 4, False)
    assert not ok and not exact
    assert b.band_compare(a, t, 64, 1, 4, True)[0]                   # statistical mode tolerates it


def test_dump_outputs_writes_float32_within_the_budget(tmp_path):
    b = _bench()
    import numpy as np
    b.DUMP_BYTES = 1 << 20
    small = np.arange(24, dtype=np.float16).reshape(2, 3, 4)
    big = np.random.RandomState(2).rand(512, 256, 4).astype(np.float16)   # 2 MiB as float32: over the budget
    b.dump_outputs(str(tmp_path / "a"), {"small": small, "big": big})
    b.dump_outputs(str(tmp_path / "b"), {"small": small, "big": big})
    s, g = np.load(tmp_path / "a" / "small.npy"), np.load(tmp_path / "a" / "big.npy")
    assert s.dtype == np.float32 and np.array_equal(s, small.astype(np.float32))
    assert g.dtype == np.float32 and g.shape[1:] == big.shape[1:] and 0 < g.shape[0] < big.shape[0]
    assert sum(os.path.getsize(p) for p in (tmp_path / "a").iterdir()) <= b.DUMP_BYTES
    assert np.array_equal(g, np.load(tmp_path / "b" / "big.npy"))     # the sample is fixed
    assert all(any(np.array_equal(r, x) for x in big.astype(np.float32)) for r in g[:8])
