"""Asset import (SURVEY §8 row N5): libkjb_asset.so (C++: glTF 2.0 -> TriangleMesh, PNG / JPEG -> RGBA8, Lanczos3 mip chains) against the
numpy restatement oracle/kj_asset.py, committed fixtures (tests/golden/gltf, made by tests/golden/make_gltf_fixtures.py), hand-computed
expectations, and the reference's own bundled glTF assets (the small ones, stored under tests/golden/reference_assets).  Bit-exact everywhere except JPEG (lossy codec:
max / mean texel error against libjpeg stated in the test)."""
import ctypes as C, glob, io, json, os, re, sys, zlib
import numpy as np, pytest
import conftest
from kajiya_b200 import asset

sys.path.insert(0, os.path.join(conftest.ROOT, "oracle"))
import kj_asset as oracle   # noqa: E402  (test infrastructure)

FIX = os.path.join(conftest.ROOT, "tests", "golden", "gltf")
REF_MESHES = os.path.join(conftest.ROOT, "tests", "golden", "reference_assets", "meshes")


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def assert_same_mesh(got, want, texel_tol=0):
    for k in ("positions", "normals", "uvs", "colors", "tangents", "material_ids", "indices"):
        assert got[k].shape == want[k].shape, (k, got[k].shape, want[k].shape)
        assert np.array_equal(bits(got[k]), bits(want[k])), (k, int((bits(got[k]) != bits(want[k])).sum()))
    assert len(got["materials"]) == len(want["materials"]) and len(got["maps"]) == len(want["maps"])
    for g, w in zip(got["materials"], want["materials"]):
        assert np.array_equal(bits(np.array(g["base_color"], np.float32)), bits(w["base_color"]))
        assert np.float32(g["roughness"]) == w["roughness"] and np.float32(g["metallic"]) == w["metallic"]
        assert np.array_equal(np.array(g["emissive"], np.float32), w["emissive"]) and g["flags"] == w["flags"] and g["maps"] == w["maps"]
        assert np.array_equal(bits(g["map_transforms"]), bits(w["map_transforms"]))
    for i, (g, w) in enumerate(zip(got["maps"], want["maps"])):
        lv = w["levels"]
        assert (g["width"], g["height"], g["mips"], g["srgb"]) == (lv[0].shape[1], lv[0].shape[0], len(lv), w["srgb"]), i
        flat = np.concatenate([l.reshape(-1) for l in lv])
        if texel_tol == 0:
            assert np.array_equal(g["texels"], flat), (i, int((g["texels"] != flat).sum()))
        else:
            assert np.abs(g["texels"].astype(int) - flat.astype(int)).max() <= texel_tol, i


# ------------------------------------------------------------------ ABI
def test_asset_library_exports_every_declared_symbol():
    assert os.path.exists(asset.ASSET_SO), "libkjb_asset.so missing: run __graft_entry__.build()"
    src = open(os.path.join(conftest.ROOT, "include", "kjb_asset.h")).read()
    names = sorted(set(re.findall(r"\b(kjb_asset_[a-z0-9_]+)\s*\(", src)))
    dll = C.CDLL(asset.ASSET_SO)
    assert len(names) == 9 and [n for n in names if not hasattr(dll, n)] == []


# ------------------------------------------------------------------ PNG / inflate
@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(FIX, "png", "*.png"))), ids=lambda p: os.path.basename(p)[:-4])
def test_png_fixture_decodes_exactly(path):
    want = np.load(path[:-4] + ".npy")
    got = asset.decode_image(open(path, "rb").read())
    assert got.shape == want.shape and np.array_equal(got, want)
    name = os.path.basename(path)
    # the oracle's decoder (PIL) agrees too for 8-bit-per-channel outputs; PIL compares a sub-byte grey tRNS key with the SCALED sample
    # (spec: the key is in the image's own bit depth), so those three files are pinned by the hand-written expectation alone
    if "16" not in name and not re.fullmatch(r"gray[124]_trns\.png", name):
        assert np.array_equal(oracle.decode_image(open(path, "rb").read()), want)


def test_png_written_by_an_independent_encoder():
    from PIL import Image
    rng = np.random.default_rng(5)
    for mode, ch in (("RGBA", 4), ("RGB", 3), ("L", 1), ("LA", 2)):
        a = rng.integers(0, 256, (45, 31, ch), dtype=np.uint8)
        buf = io.BytesIO(); Image.fromarray(a[..., 0] if ch == 1 else a, mode).save(buf, "PNG", optimize=True)
        assert np.array_equal(asset.decode_image(buf.getvalue()), np.asarray(Image.open(io.BytesIO(buf.getvalue())).convert("RGBA")))
    big = (np.add.outer(np.arange(700), np.arange(900)) // 3 % 256).astype(np.uint8)   # long matches, several deflate blocks
    buf = io.BytesIO(); Image.fromarray(big, "L").save(buf, "PNG")
    assert np.array_equal(asset.decode_image(buf.getvalue())[..., 0], big)


def test_png_errors_are_reported():
    good = open(os.path.join(FIX, "png", "rgba8.png"), "rb").read()
    bad_crc = bytearray(good); bad_crc[40] ^= 0x55
    for data, msg in ((bytes(bad_crc), "CRC"), (good[:60], "png"), (b"GIF89a" + bytes(32), "unrecognised"), (good[:8] + good[33:], "IHDR")):
        with pytest.raises(asset.AssetError, match=msg):
            asset.decode_image(data)
    # corrupt the zlib stream but keep chunk CRCs valid
    import struct
    pos = good.index(b"IDAT"); ln = struct.unpack(">I", good[pos - 4:pos])[0]
    body = bytearray(good[pos + 4:pos + 4 + ln]); body[len(body) // 2] ^= 0xff
    broken = good[:pos + 4] + bytes(body) + struct.pack(">I", zlib.crc32(b"IDAT" + bytes(body)) & 0xffffffff) + good[pos + 8 + ln:]
    with pytest.raises(asset.AssetError, match="corrupt image data"):
        asset.decode_image(broken)


# ------------------------------------------------------------------ JPEG
@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(FIX, "jpg", "*.jpg"))), ids=lambda p: os.path.basename(p)[:-4])
def test_jpeg_fixture_against_libjpeg(path):
    """Lossy codec: decoders legitimately differ in IDCT rounding and chroma upsampling taps.  Tolerance: every channel within 3/255 of
    libjpeg-turbo's output (PIL), mean absolute error below 0.25/255; greyscale (no upsampling, no colour transform) within 1/255."""
    got = asset.decode_image(open(path, "rb").read()).astype(int)
    want = oracle.decode_image(open(path, "rb").read()).astype(int)
    assert got.shape == want.shape and (got[..., 3] == 255).all()
    err = np.abs(got - want)
    if "gray" in os.path.basename(path):
        assert err.max() <= 1 and (got[..., 0] == got[..., 1]).all()
    else:
        assert err.max() <= 3 and err.mean() < 0.25, (err.max(), err.mean())


def test_jpeg_errors_are_reported():
    good = open(os.path.join(FIX, "jpg", "baseline_420.jpg"), "rb").read()
    with pytest.raises(asset.AssetError, match="jpeg"):
        asset.decode_image(good[:200])
    with pytest.raises(asset.AssetError, match="jpeg"):
        asset.decode_image(b"\xff\xd8\xff\xd9")


# ------------------------------------------------------------------ DDS
def _dds(dxgi, w, h, mips, seed):
    import struct
    rng = np.random.default_rng(seed)
    bb = 8 if dxgi == 72 else 16
    body = b""
    for l in range(mips):
        lw, lh = max(1, w >> l), max(1, h >> l)
        body += rng.integers(0, 256, ((max(lw, 4) + 3) // 4) * ((max(lh, 4) + 3) // 4) * bb, dtype=np.uint8).tobytes()   # any bytes are valid BC blocks
    hdr = struct.pack("<4sIIIIIII44x", b"DDS ", 124, 0x1007 | 0x20000, h, w, 0, 0, mips) + struct.pack("<II4sIIIII", 32, 4, b"DX10", 0, 0, 0, 0, 0) + struct.pack("<IIIII", 0x1000 | 0x400000, 0, 0, 0, 0)
    return hdr + struct.pack("<IIIII", dxgi, 3, 0, 1, 0) + body


@pytest.mark.parametrize("dxgi,w,h,mips", [(72, 16, 12, 5), (77, 20, 20, 3), (78, 8, 8, 4), (83, 13, 7, 1), (84, 32, 4, 6)])
def test_dds_block_decoding_matches_the_restatement(dxgi, w, h, mips):
    """process_dds accepts BC1_SRGB / BC3 / BC3_SRGB / BC5 / BC5_SNORM with their own mip chains; random blocks, odd extents, sub-block mips"""
    data = _dds(dxgi, w, h, mips, dxgi * 100 + w)
    want, srgb = oracle.decode_dds(data)
    top = asset.decode_image(data)
    assert top.shape == want[0].shape and np.array_equal(top, want[0])
    assert len(want) == mips and [l.shape[:2] for l in want] == [(max(1, h >> l), max(1, w >> l)) for l in range(mips)] and srgb == (1 if dxgi in (72, 78) else 0)


def test_dds_hand_decoded_blocks():
    import struct
    def file(dxgi, block):
        hdr = struct.pack("<4sIIIIIII44x", b"DDS ", 124, 0x1007, 4, 4, 0, 0, 1) + struct.pack("<II4sIIIII", 32, 4, b"DX10", 0, 0, 0, 0, 0) + struct.pack("<IIIII", 0x1000, 0, 0, 0, 0)
        return hdr + struct.pack("<IIIII", dxgi, 3, 0, 1, 0) + block
    # BC1: c0 = pure red (0xF800) > c1 = pure blue (0x001F): four-colour mode; indices 0,1,2,3 repeating
    img = asset.decode_image(file(72, struct.pack("<HHI", 0xF800, 0x001F, 0xE4E4E4E4)))
    assert [tuple(int(v) for v in img[0, x]) for x in range(4)] == [(255, 0, 0, 255), (0, 0, 255, 255), (170, 0, 85, 255), (85, 0, 170, 255)]
    # c0 <= c1: three colours + transparent black
    img = asset.decode_image(file(72, struct.pack("<HHI", 0x001F, 0xF800, 0xE4E4E4E4)))
    assert tuple(int(v) for v in img[0, 2]) == (127, 0, 127, 255) and tuple(int(v) for v in img[0, 3]) == (0, 0, 0, 0)
    # BC5_UNORM: red ramp 255 > 0 (six interpolants), green 0 < 255 (four interpolants + 0 and 1)
    red = bytes([255, 0]) + (0o76543210 | (0o76543210 << 24)).to_bytes(6, "little"); green = bytes([0, 255]) + (0o76543210 | (0o76543210 << 24)).to_bytes(6, "little")
    img = asset.decode_image(file(83, red + green))
    assert [int(v) for v in img.reshape(-1, 4)[:8, 0]] == [255, 0, 219, 182, 146, 109, 73, 36]
    assert [int(v) for v in img.reshape(-1, 4)[:8, 1]] == [0, 255, 51, 102, 153, 204, 0, 255]
    for bad, msg in ((b"DDS " + bytes(200), "bad header"), (file(71, bytes(8)), "not supported"), (file(72, bytes(4)), "past the end")):
        with pytest.raises(asset.AssetError, match=msg):
            asset.decode_image(bad)


def test_gltf_with_dds_textures_uses_the_files_own_mips(tmp_path):
    import shutil
    doc = json.load(open(os.path.join(FIX, "courtyard.gltf")))
    for f in ("courtyard.bin", "spec.png"):
        shutil.copy(os.path.join(FIX, f), tmp_path)
    (tmp_path / "albedo.dds").write_bytes(_dds(72, 16, 8, 5, 7))
    doc["images"][0] = {"uri": "albedo.dds"}
    (tmp_path / "dds.gltf").write_text(json.dumps(doc))
    sc = asset.GltfScene(str(tmp_path / "dds.gltf")); a = sc.arrays()
    assert_same_mesh(a, oracle.load_gltf_scene(str(tmp_path / "dds.gltf")))
    m = a["maps"][2]
    assert (m["width"], m["height"], m["mips"], m["srgb"]) == (16, 8, 5, 1)     # the file's chain and its sRGB format, not TexParams / Lanczos


# ------------------------------------------------------------------ mip chains
@pytest.mark.parametrize("w,h", [(37, 21), (64, 64), (1, 9), (5, 1), (130, 7)])
def test_mip_chain_matches_the_restatement(w, h):
    rng = np.random.default_rng(w * 1000 + h)
    img = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    levels, ow, oh = asset.build_mips(img)
    want = oracle.process_rgba8(img)
    assert (ow, oh) == (w, h) and len(levels) == len(want) == max(w.bit_length(), h.bit_length())   # mip_count_1d: floor(log2) + 1
    for l, (g, wnt) in enumerate(zip(levels, want)):
        assert g.shape == (max(1, h >> l), max(1, w >> l), 4) and np.array_equal(g, wnt), l
    assert np.array_equal(levels[0], img)


def test_mip_chain_properties():
    flat = np.full((40, 24, 4), 93, np.uint8)
    for l in asset.build_mips(flat)[0]:   # weights are normalised: a constant image stays constant at every level
        assert (l == 93).all()
    img = np.random.default_rng(1).integers(0, 256, (16, 16, 4), dtype=np.uint8)
    plain = asset.build_mips(img)[0]
    swz = asset.build_mips(img, swizzle=[1, 2, 0, 3])[0]
    for p, s in zip(plain, swz):   # image.rs:214-223 writes the channels in place one by one: (g, b, g, a); levels are resampled before the swizzle
        assert np.array_equal(s[..., 0], p[..., 1]) and np.array_equal(s[..., 1], p[..., 2]) and np.array_equal(s[..., 2], p[..., 1]) and np.array_equal(s[..., 3], p[..., 3])
    only, w, h = asset.build_mips(img, use_mips=False)
    assert len(only) == 1 and np.array_equal(only[0], img)


def test_oversized_images_are_clamped_to_2048():
    img = np.random.default_rng(2).integers(0, 256, (3, 2100, 4), dtype=np.uint8)
    levels, w, h = asset.build_mips(img)
    want = oracle.process_rgba8(img)
    assert (w, h) == (2048, 3) and len(levels) == 12 and all(np.array_equal(a, b) for a, b in zip(levels, want))


# ------------------------------------------------------------------ glTF
@pytest.mark.parametrize("name", ["courtyard.gltf", "courtyard.glb"])
def test_courtyard_matches_the_restatement(name):
    path = os.path.join(FIX, name)
    sc = asset.GltfScene(path)
    assert_same_mesh(sc.arrays(), oracle.load_gltf_scene(path))
    assert sc.stats == dict(nodes=8, primitives=7, skipped=1, images=3)


def test_courtyard_semantics():
    a = asset.GltfScene(os.path.join(FIX, "courtyard.gltf")).arrays()
    b = asset.GltfScene(os.path.join(FIX, "courtyard.glb")).arrays()
    for k in ("positions", "normals", "uvs", "colors", "tangents", "material_ids", "indices"):
        assert np.array_equal(bits(a[k]), bits(b[k])), k            # the container does not matter
    # traversal order: root{floor(grid, fan), mirrored(cube){broken(1 kept, then the node is left)}, rig{leaf}}, floor again(grid, fan), sparse
    counts = [25, 6, 24, 6, 25, 6, 6]
    assert len(a["positions"]) == sum(counts)
    # one material + four maps per visited primitive, including the one without NORMAL (pushed before the early return)
    assert len(a["materials"]) == 8 and len(a["maps"]) == 32
    assert [m["maps"] for m in a["materials"]] == [[4 * i + k for k in range(4)] for i in range(8)]
    assert np.array_equal(a["material_ids"], np.repeat([0, 1, 2, 3, 5, 6, 7], counts).astype(np.uint32))   # material 4 has no vertices, 7 is the default one
    # indices are rebased per primitive and stay inside it
    start = np.cumsum([0] + counts)
    ic = [96, 6, 36, 6, 96, 6, 6]; istart = np.cumsum([0] + ic)
    for p in range(7):
        seg = a["indices"][istart[p]:istart[p + 1]]
        assert seg.min() >= start[p] and seg.max() < start[p + 1]
    # the mirrored node has a negative determinant: winding reversed, tangent handedness negated
    cube = a["indices"][istart[2]:istart[3]].reshape(-1, 3) - start[2]
    assert np.array_equal(cube[0], [2, 1, 0]) and np.array_equal(cube[1], [3, 2, 0])
    tw = a["tangents"][start[2]:start[3], 3]
    assert np.array_equal(tw, np.where(np.arange(24) % 2 == 0, -1.0, 1.0).astype(np.float32))
    # no TANGENT attribute: the (1,0,0,0) default goes through the node transform like a real tangent, its zero handedness survives
    assert (a["tangents"][:25, 3] == 0).all() and np.allclose(np.linalg.norm(a["tangents"][:25, :3], axis=1), 1.0, atol=1e-6) and (a["tangents"][:25] == a["tangents"][0]).all()
    # geometry facts that do not depend on float rounding
    assert np.allclose(np.linalg.norm(a["normals"], axis=1), 1.0, atol=1e-6)
    assert np.allclose(a["positions"][start[6] + 1], np.array([1, 0.9, 0]) + [-2, 0.5, 0], atol=1e-6)    # sparse substitution, then the node translation
    assert np.allclose(a["positions"][start[6] + 0], np.array([0, 0.5, 0]) + [-2, 0.5, 0], atol=1e-6)
    # normalised integer attributes
    assert a["uvs"][:25].min() == 0.0 and a["uvs"][:25].max() == 1.0 and np.allclose(a["uvs"][1], [0.25, 0.0], atol=1e-5)
    assert (a["colors"][:25] <= 1.0).all() and (a["colors"][25:31, 3] == 1.0).all() and (a["colors"][31:55] == 1.0).all()
    # materials
    m0, m2, m8 = a["materials"][0], a["materials"][2], a["materials"][7]
    assert np.allclose(m0["base_color"], [0.9, 0.8, 0.7, 1.0]) and np.isclose(m0["roughness"], 0.85) and np.isclose(m0["metallic"], 0.25)
    c, s = np.cos(0.4), np.sin(0.4)
    assert np.allclose(m0["map_transforms"][0], [c * 3, s * 2, -s * 3, c * 2, 0.125, 0.25], atol=1e-6)
    assert np.array_equal(m0["map_transforms"][1:], np.tile(np.array([1, 0, 0, 1, 0, 0], np.float32), (3, 1)))
    assert m8["base_color"] == [1, 1, 1, 1] and m8["roughness"] == 1.0 and m8["metallic"] == 1.0 and m8["emissive"] == [0, 0, 0]
    assert m2["emissive"] == [2.0, 1.5, 0.5] and np.isclose(m2["roughness"], 0.3)
    maps = a["maps"]
    # placeholders (1x1, linear): normal (127,127,255,255), spec (255,255,127,255), albedo / emissive white
    assert [list(maps[4 + k]["texels"]) for k in range(4)] == [[127, 127, 255, 255], [255, 255, 127, 255], [255, 255, 255, 255], [255, 255, 255, 255]]
    assert all(maps[4 + k]["srgb"] == 0 and maps[4 + k]["mips"] == 1 for k in range(4))
    # image maps: albedo 37x21 sRGB with 6 levels, spec 16x16 linear swizzled, emissive 8x8 sRGB from the data: URI palette PNG, normal linear
    assert (maps[2]["width"], maps[2]["height"], maps[2]["mips"], maps[2]["srgb"]) == (37, 21, 6, 1)
    assert (maps[1]["width"], maps[1]["height"], maps[1]["mips"], maps[1]["srgb"]) == (16, 16, 5, 0)
    assert (maps[11]["width"], maps[11]["height"], maps[11]["mips"], maps[11]["srgb"]) == (8, 8, 4, 1)
    assert (maps[8]["width"], maps[8]["srgb"]) == (16, 0)
    from PIL import Image
    spec = np.asarray(Image.open(os.path.join(FIX, "spec.png")).convert("RGBA"))
    lvl0 = maps[1]["texels"][:16 * 16 * 4].reshape(16, 16, 4)
    assert np.array_equal(lvl0[..., 0], spec[..., 1]) and np.array_equal(lvl0[..., 1], spec[..., 2]) and np.array_equal(lvl0[..., 2], spec[..., 1])
    assert np.array_equal(maps[8]["texels"][:16 * 16 * 4].reshape(16, 16, 4), spec)    # the same image as a normal map: unswizzled
    assert np.array_equal(maps[12 + 2]["texels"], maps[2]["texels"])                    # KHR_materials_pbrSpecularGlossiness.diffuseTexture fallback


def test_root_transform_scale_and_rotation():
    path = os.path.join(FIX, "courtyard.gltf")
    q = (0.0, float(np.sin(0.35)), 0.0, float(np.cos(0.35)))
    a = asset.GltfScene(path, scale=2.5, rotation=q).arrays()
    assert_same_mesh(a, oracle.load_gltf_scene(path, 2.5, q))
    base = asset.GltfScene(path).arrays()
    ang = 0.7; R = np.array([[np.cos(ang), 0, np.sin(ang)], [0, 1, 0], [-np.sin(ang), 0, np.cos(ang)]])
    assert np.allclose(a["positions"], 2.5 * base["positions"] @ R.T, atol=2e-5) and np.allclose(a["normals"], base["normals"] @ R.T, atol=1e-5)
    assert np.array_equal(a["indices"], base["indices"])


def test_gltf_errors_are_reported(tmp_path):
    doc = json.load(open(os.path.join(FIX, "courtyard.gltf")))

    def attempt(mutate, msg, raw=None):
        d = json.loads(json.dumps(doc)); mutate(d)
        p = tmp_path / "case.gltf"
        p.write_text(raw if raw is not None else json.dumps(d))
        for f in ("courtyard.bin", "albedo tex.png", "spec.png"):
            if not (tmp_path / f).exists():
                (tmp_path / f).write_bytes(open(os.path.join(FIX, f), "rb").read())
        with pytest.raises(asset.AssetError, match=msg):
            asset.GltfScene(str(p))
    with pytest.raises(asset.AssetError, match="cannot open"):
        asset.GltfScene(str(tmp_path / "missing.gltf"))
    attempt(lambda d: None, "gltf: ", raw='{"asset": {"version": "2.0"}, "scenes": [')
    attempt(lambda d: d.pop("scenes"), "No default scene")
    attempt(lambda d: d["buffers"][0].update(uri="nope.bin"), "cannot open")
    attempt(lambda d: d["buffers"][0].update(uri="ftp://host/x.bin"), "unsupported URI scheme")
    attempt(lambda d: d["buffers"][0].update(byteLength=10 ** 7), "document says")
    attempt(lambda d: d["accessors"][0].update(count=10 ** 6), "past its buffer view")
    attempt(lambda d: d["meshes"][1]["primitives"][0].update(indices=0), "index out of range|SCALAR|bad")
    attempt(lambda d: d["images"][0].update(uri="spec.pn"), "cannot open")
    attempt(lambda d: d["meshes"][0]["primitives"][1].update(mode=5), "triangle lists")
    attempt(lambda d: d["scenes"][1].update(nodes=[99]), "unknown node")
    glb = open(os.path.join(FIX, "courtyard.glb"), "rb").read()
    (tmp_path / "cut.glb").write_bytes(glb[:len(glb) // 2])
    with pytest.raises(asset.AssetError, match="glb"):
        asset.GltfScene(str(tmp_path / "cut.glb"))


def test_json_parser_corner_cases(tmp_path):
    """escapes, surrogate pairs, exponents, a byte order mark, nesting, and things that must be rejected"""
    doc = {"asset": {"version": "2.0", "copyright": "café 🚀 \"quoted\" \\ / \b\f\n\r\t"}, "scene": 0, "scenes": [{"nodes": [0]}],
           "nodes": [{"name": "n", "translation": [1e0, -2.5E-1, 3.0e+0]}]}
    p = tmp_path / "bom.gltf"; p.write_bytes(b"\xef\xbb\xbf" + json.dumps(doc, ensure_ascii=True).encode())
    assert asset.GltfScene(str(p)).stats["nodes"] == 1
    for bad in ('{"a": 01}', '{"a": [1,]}', '{"a": "\\x"}', '{"a": tru}', '{"a": 1} x', '["' + "[" * 400 + '"]', '{"a": "unterminated}'):
        q = tmp_path / "bad.gltf"; q.write_text(bad)
        with pytest.raises(asset.AssetError):
            asset.GltfScene(str(q))


# ------------------------------------------------------------------ the reference's own bundled assets
REF_CASES = [("cornell_box/scene.gltf", 0), ("floor/scene.gltf", 0), ("roughness-scale/scene.gltf", 0), ("emissive/triangle.glb", 0),
             ("conference_jake/scene.gltf", 8)]   # the textured node of the reference's conference scene (tests/golden/make_reference_subsets.py)


@pytest.mark.parametrize("rel,texel_tol", REF_CASES, ids=[c[0].split("/")[0] for c in REF_CASES])
def test_reference_assets_match_the_restatement(rel, texel_tol):
    """conference_jake carries a JPEG: its maps are compared within 8/255 (decoder + resampling of decoder differences), everything else exactly"""
    path = os.path.join(REF_MESHES, rel)
    assert_same_mesh(asset.GltfScene(path).arrays(), oracle.load_gltf_scene(path), texel_tol)


def test_bundled_cornell_box_fixture_is_the_reference_asset():
    """kajiya_b200/assets/cornell_box.json (the bench scene, baked in float64 by tests/golden/make_assets.py) is the same mesh the importer
    produces from the reference's scene.gltf: identical topology and materials, vertices within one float32 ulp of the f32 transform chain."""
    a = asset.GltfScene(os.path.join(REF_MESHES, "cornell_box/scene.gltf")).arrays()
    j = json.load(open(os.path.join(conftest.ROOT, "kajiya_b200", "assets", "cornell_box.json")))
    assert np.array_equal(a["indices"], np.array(j["indices"], np.uint32)) and np.array_equal(a["material_ids"], np.array(j["material_ids"], np.uint32))
    assert np.abs(a["positions"] - np.array(j["positions"], np.float32)).max() <= 2.4e-7 and np.abs(a["normals"] - np.array(j["normals"], np.float32)).max() <= 2.4e-7
    for m, jm in zip(a["materials"], j["materials"]):
        assert np.allclose(m["base_color"], jm["base_color"]) and np.isclose(m["roughness"], jm["roughness"]) and np.isclose(m["metallic"], jm["metallic"])


# ------------------------------------------------------------------ importer -> add_mesh -> frames
def _courtyard_world(lib, **kw):
    import parity
    from kajiya_b200 import scenes
    from kajiya_b200.world import World
    sc = asset.GltfScene(os.path.join(FIX, "courtyard.gltf"))
    w = World(lib, 72, 48, **kw)
    h = w.add_mesh_desc(sc.desc)
    w.add_instance(h, np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]], np.float32))
    w.set_blue_noise(scenes.blue_noise()); w.set_spatial_resolve_offsets(scenes.spatial_resolve_offsets())
    sc.close()   # add_mesh copied everything it needs
    return w


COURTYARD_VIEW = dict(camera_position=(0.5, 2.5, 7.0), camera_rotation=(float(np.sin(-0.15)), 0.0, 0.0, float(np.cos(-0.15))), sun_direction=(0.35, 0.8, 0.45))


def test_imported_scene_renders_identically_on_oracle_and_emulator(oracle_lib, emu_lib):
    """the importer's kjb_mesh_desc goes straight into add_mesh; textured, texture-transformed, vertex-coloured, emissive-mapped hits are
    shaded by the kernels and by the oracle from the same texels: every image of every frame bit-for-bit"""
    import parity
    kw = dict(enable_rtr=True, enable_lighting=True)
    wa, wb = _courtyard_world(oracle_lib, **kw), _courtyard_world(emu_lib, **kw)
    for f in range(3):
        wa.render_frame(**COURTYARD_VIEW); wb.render_frame(**COURTYARD_VIEW)
        assert not parity.compare_images(wa, wb), f
    gb = wb.image("gbuffer")
    assert (wb.image("depth") > 0).mean() > 0.25            # the scene is in view
    albedo_words = np.unique(gb[..., 0].view(np.uint32))
    assert len(albedo_words) > 200                            # the albedo map + vertex colours vary across the floor (a flat material would give a handful)


@pytest.mark.gpu
def test_imported_scene_renders_identically_on_gpu(oracle_lib, cuda_lib):
    import parity
    kw = dict(enable_rtr=True, enable_lighting=True)
    wa, wb = _courtyard_world(oracle_lib, **kw), _courtyard_world(cuda_lib, **kw)
    for f in range(3):
        wa.render_frame(**COURTYARD_VIEW); wb.render_frame(**COURTYARD_VIEW)
        assert not parity.compare_images(wa, wb), f


# ------------------------------------------------------------------ robustness: malformed inputs are errors, never crashes
_FUZZ = r'''
import sys, os, glob, random, struct, zlib, json, shutil
sys.path.insert(0, sys.argv[1])
from kajiya_b200 import asset
fix, tmp = sys.argv[2], sys.argv[3]
random.seed(1234)
def refix(d):   # recompute chunk CRCs so that mutations reach the inflater and the unfilter / expand code
    out = bytearray(d[:8]); off = 8
    while off + 12 <= len(d):
        ln = struct.unpack(">I", d[off:off + 4])[0]; typ = d[off + 4:off + 8]; body = d[off + 8:off + 8 + ln]
        if off + 12 + ln > len(d): out += d[off:]; break
        out += d[off:off + 8] + body + struct.pack(">I", zlib.crc32(typ + body) & 0xffffffff); off += 12 + ln
    return bytes(out)
images = sorted(glob.glob(os.path.join(fix, "png", "*.png")))[::5] + sorted(glob.glob(os.path.join(fix, "jpg", "*.jpg")))
decoded = rejected = 0
for it in range(700):
    f = random.choice(images); d = bytearray(open(f, "rb").read()); r = random.random()
    if r < 0.6:
        for _ in range(random.randint(1, 5)): d[random.randrange(8, len(d))] = random.randrange(256)
    elif r < 0.8: d = d[:random.randrange(1, len(d))]
    else: i = random.randrange(len(d)); d[i:i] = bytes(random.randrange(256) for _ in range(random.randint(1, 30)))
    data = refix(bytes(d)) if f.endswith(".png") and random.random() < 0.7 else bytes(d)
    try: asset.decode_image(data); decoded += 1
    except asset.AssetError: rejected += 1
for f in ("courtyard.bin", "albedo tex.png", "spec.png"): shutil.copy(os.path.join(fix, f), tmp)
doc = json.load(open(os.path.join(fix, "courtyard.gltf")))
def mutate(o):
    if isinstance(o, dict):
        k = random.choice(list(o.keys()))
        if random.random() < 0.15: o.pop(k); return
        if isinstance(o[k], (dict, list)) and o[k]: mutate(o[k])
        else: o[k] = random.choice([-1, 0, 1, 2 ** 31, 10 ** 9, 3.5, "x", None, [], {}, True, 65536, 5126, 5121])
    elif isinstance(o, list):
        i = random.randrange(len(o))
        if isinstance(o[i], (dict, list)) and o[i]: mutate(o[i])
        else: o[i] = random.choice([-1, 0, 1, 2 ** 31, 10 ** 9, 3.5, "x", None, [], {}, 99999])
loaded = refused = 0
for it in range(500):
    d = json.loads(json.dumps(doc))
    for _ in range(random.randint(1, 3)): mutate(d)
    open(os.path.join(tmp, "m.gltf"), "w").write(json.dumps(d))
    try: s = asset.GltfScene(os.path.join(tmp, "m.gltf")); s.arrays(); s.close(); loaded += 1
    except asset.AssetError: refused += 1
print("FUZZ", decoded, rejected, loaded, refused)
'''


def test_malformed_inputs_never_crash_the_importer(tmp_path):
    """700 mutated PNG/JPEG streams (chunk CRCs repaired so the damage reaches the decoders) and 500 mutated glTF documents, in a child
    process so that an abort or a segfault would be seen: every input either decodes or is refused with an error"""
    import subprocess
    r = subprocess.run([sys.executable, "-c", _FUZZ, conftest.ROOT, FIX, str(tmp_path)], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=600)
    assert r.returncode == 0, (r.returncode, r.stderr[-500:])
    tag, decoded, rejected, loaded, refused = r.stdout.split()[-5:]
    assert tag == "FUZZ" and int(decoded) + int(rejected) == 700 and int(loaded) + int(refused) == 500 and int(rejected) > 100 and int(refused) > 100


# ------------------------------------------------------------------ structured hostile inputs, against an ASan + UBSan build of the importer
_HOSTILE = r'''
import sys, os, json, struct, shutil
sys.path.insert(0, sys.argv[1])
from kajiya_b200 import asset
fix, tmp = sys.argv[2], sys.argv[3]
for f in ("courtyard.bin", "albedo tex.png", "spec.png"): shutil.copy(os.path.join(fix, f), tmp)
doc = json.load(open(os.path.join(fix, "courtyard.gltf")))
def with_(path, value):
    d = json.loads(json.dumps(doc)); o = d
    for k in path[:-1]: o = o[k]
    o[path[-1]] = value
    return d
acc_with_view = next(i for i, a in enumerate(doc["accessors"]) if "bufferView" in a)
bv = doc["accessors"][acc_with_view]["bufferView"]
cases = []
for v in (4611686018427387904, 2 ** 63, 2 ** 64, 1e300, -1, -16, 2.5, 2 ** 53, 2 ** 40):
    cases.append(with_(["accessors", acc_with_view, "count"], v))
    cases.append(with_(["accessors", acc_with_view, "byteOffset"], v))
    cases.append(with_(["bufferViews", bv, "byteOffset"], v))
    cases.append(with_(["bufferViews", bv, "byteLength"], v))
    cases.append(with_(["bufferViews", bv, "byteStride"], v))
    cases.append(with_(["buffers", 0, "byteLength"], v))
d = with_(["accessors", acc_with_view, "count"], 4611686018427387904); d["accessors"][acc_with_view]["type"] = "VEC4"; d["bufferViews"][bv]["byteStride"] = 16; cases.append(d)
for v in (4611686018427387904, -1, 2 ** 32, 10 ** 6):
    d = json.loads(json.dumps(doc)); a = d["accessors"][acc_with_view]
    a["sparse"] = {"count": v, "indices": {"bufferView": bv, "componentType": 5125, "byteOffset": 0}, "values": {"bufferView": bv, "byteOffset": 0}}; cases.append(d)
    d = json.loads(json.dumps(doc)); a = d["accessors"][acc_with_view]
    a["sparse"] = {"count": 1, "indices": {"bufferView": bv, "componentType": 5125, "byteOffset": v}, "values": {"bufferView": bv, "byteOffset": v}}; cases.append(d)
if doc.get("images"):
    for v in (-16, 2 ** 63, 2 ** 64 - 8):
        d = json.loads(json.dumps(doc)); d["images"][0] = {"bufferView": bv, "mimeType": "image/png"}; d["bufferViews"][bv]["byteOffset"] = v; cases.append(d)
        d = json.loads(json.dumps(doc)); d["images"][0] = {"bufferView": -1, "mimeType": "image/png"}; cases.append(d)
loaded = refused = 0
for d in cases:
    open(os.path.join(tmp, "h.gltf"), "w").write(json.dumps(d))
    try: s = asset.GltfScene(os.path.join(tmp, "h.gltf")); s.arrays(); s.close(); loaded += 1
    except asset.AssetError: refused += 1
good = open(os.path.join(fix, "jpg", "baseline_420.jpg"), "rb").read()
sos = good.index(b"\xff\xda")
jpegs = [good[:sos] + b"\xff\xda\x00\x02", good[:sos] + b"\xff\xda\x00\x03\x03", b"\xff\xd8\xff\xda\x00\x02"]
sof = good.index(b"\xff\xc0")
big = bytearray(good); big[sof + 5:sof + 9] = b"\xff\xff\xff\xff"; jpegs.append(bytes(big[:sos + 40]))
dqt = good.index(b"\xff\xdb")
q16 = bytearray(good[:dqt]) + b"\xff\xdb" + struct.pack(">H", 2 + 129) + bytes([0x10]) + b"\xff\xff" * 64 + good[dqt:]   # a 16-bit table 0 of 65535s ahead of the real ones ...
jpegs.append(bytes(q16))
ln = struct.unpack(">H", good[dqt + 2:dqt + 4])[0]
q16b = bytearray(good[:dqt + 2 + ln]) + b"\xff\xdb" + struct.pack(">H", 2 + 129) + bytes([0x10]) + b"\xff\xff" * 64 + good[dqt + 2 + ln:]   # ... and one that replaces table 0 before the scan
jpegs.append(bytes(q16b))
dec = rej = 0
for j in jpegs:
    try: asset.decode_image(j); dec += 1
    except asset.AssetError: rej += 1
print("HOSTILE", len(cases), loaded, refused, len(jpegs), dec, rej)
'''


def test_structured_hostile_inputs_under_sanitizers(tmp_path):
    """Numeric-field overflows (count / byteOffset / byteStride / byteLength at 2^62, 2^64, negative, fractional; sparse views; image buffer
    views), a SOS cut after its length word, a 65535^2 SOF on a tiny file and 16-bit quantisation tables of 65535 — against the importer
    built with AddressSanitizer + UBSan, in a child process: every case is refused or decodes, and the sanitizers stay silent"""
    import shutil, subprocess
    if not shutil.which("g++"):
        pytest.skip("no host compiler")
    host = os.path.join(conftest.ROOT, "kajiya_b200", "csrc", "host")
    out = os.path.join(conftest.ROOT, "tests", "emu", "_build_san", "libkjb_asset_san.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    srcs = [os.path.join(host, f) for f in ("kjb_asset.cpp", "kjb_asset_image.cpp")]
    deps = srcs + [os.path.join(host, "kjb_asset_json.h")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-fno-omit-frame-pointer", "-fsanitize=address,undefined",
                        "-fno-sanitize=vptr", "-fno-sanitize-recover=undefined", "-I", os.path.join(conftest.ROOT, "include")] + srcs + ["-o", out], check=True)
    rt = subprocess.run(["gcc", "-print-file-name=libasan.so"], stdout=subprocess.PIPE, text=True).stdout.strip()
    env = dict(os.environ, KJB_ASSET_SO=out, LD_PRELOAD=rt, ASAN_OPTIONS="detect_leaks=0:halt_on_error=1:abort_on_error=1", UBSAN_OPTIONS="halt_on_error=1:print_stacktrace=1")
    r = subprocess.run([sys.executable, "-c", _HOSTILE, conftest.ROOT, FIX, str(tmp_path)], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=600, env=env)
    assert r.returncode == 0, (r.returncode, r.stderr[-1500:])
    assert "ERROR: AddressSanitizer" not in r.stderr and "runtime error" not in r.stderr, r.stderr[-1500:]
    tag, ncases, loaded, refused, njpeg, dec, rej = r.stdout.split()[-7:]
    assert tag == "HOSTILE" and int(loaded) + int(refused) == int(ncases) and int(refused) >= int(ncases) - 12 and int(dec) + int(rej) == int(njpeg) and int(rej) >= 4
