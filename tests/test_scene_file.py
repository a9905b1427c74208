"""kajiya scene files (.ron) -> instances (kajiya_b200/scene_file.py; mirrors crates/bin/view/src/{scene,runtime,persisted}.rs)."""
import glob, os
import numpy as np, pytest
import conftest
from kajiya_b200 import scene_file, scenes
from kajiya_b200.world import World

GOLDEN = os.path.join(conftest.ROOT, "tests", "golden")
REF_ASSETS = os.path.join(GOLDEN, "reference_assets")   # the reference's scene files and the meshes the Cornell box scene names
REF_SCENES = os.path.join(REF_ASSETS, "scenes")


def test_parse_fixture_and_defaults():
    inst = scene_file.read_scene(os.path.join(GOLDEN, "scene_fixture.ron"))
    assert [i["mesh"] for i in inst] == ["/gltf/courtyard.gltf"] * 2
    assert inst[0] == dict(mesh="/gltf/courtyard.gltf", position=[0.0, -1.0, 0.0], rotation=[0.0, 0.0, 0.0], scale=[2.0, 2.0, 2.0])
    assert inst[1]["scale"] == [1.0, 1.0, 1.0] and inst[1]["rotation"] == [0.0, 90.0, 0.0] and inst[1]["position"] == [1.5, 0.25, -3.0]


def test_ron_subset():
    v = scene_file.parse_ron('Foo( a: [1, 2.5, -3e2,], b: "x\\"y", c: (true, false), d: Bar(1), e: (), /* c */ f: ( g: 1 ), ) // end')
    assert v == dict(a=[1, 2.5, -300.0], b='x"y', c=[True, False], d=[1], e=[], f=dict(g=1))
    for bad in ("(instances: [", "(a: 1 b: 2)", "(a: @)", "(a: 1) x"):
        with pytest.raises(scene_file.RonError):
            scene_file.parse_ron(bad)


def test_affine_transform():
    m = scene_file.instance_transform((0, -1, 0), scale=(2, 2, 2))
    assert np.array_equal(m, np.array([[2, 0, 0, 0], [0, 2, 0, -1], [0, 0, 2, 0]], np.float32))          # assets/scenes/cornell_box.ron
    m = scene_file.instance_transform((1, 2, 3), (0, 90, 0), (1, 1, 1))                                   # +90 deg about Y: x -> -z, z -> x
    assert np.allclose(m, [[0, 0, 1, 1], [0, 1, 0, 2], [-1, 0, 0, 3]], atol=1e-6)
    # YXZ order: R = Ry * Rx * Rz
    def R(axis, deg):
        a = np.radians(deg); c, s = np.cos(a), np.sin(a)
        return {"x": np.array([[1, 0, 0], [0, c, -s], [0, s, c]]), "y": np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]]), "z": np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])}[axis]
    m = scene_file.instance_transform((0, 0, 0), (20, 35, -50), (1.5, 0.5, 2.0))
    assert np.allclose(m[:, :3], R("y", 35) @ R("x", 20) @ R("z", -50) @ np.diag([1.5, 0.5, 2.0]), atol=1e-6)


def test_load_scene_on_a_world(oracle_lib, emu_lib):
    """both instances of the fixture scene end up in the acceleration structure: the frame renders bit for bit on oracle and emulator"""
    import parity
    worlds = []
    for lib in (oracle_lib, emu_lib):
        w = World(lib, 64, 40)
        handles = scene_file.load_scene(w, os.path.join(GOLDEN, "scene_fixture.ron"), GOLDEN)
        assert len(handles) == 2
        w.set_blue_noise(scenes.blue_noise()); worlds.append(w)
    view = dict(camera_position=(0.5, 3.0, 11.0), camera_rotation=(float(np.sin(-0.1)), 0.0, 0.0, float(np.cos(-0.1))), sun_direction=(0.35, 0.8, 0.45))
    for f in range(3):
        for w in worlds: w.render_frame(**view)
        assert not parity.compare_images(*worlds), f
    assert (worlds[1].image("depth") > 0).mean() > 0.1


def test_reference_scene_files_parse():
    files = sorted(glob.glob(os.path.join(REF_SCENES, "*.ron")))
    assert len(files) >= 9
    for f in files:
        inst = scene_file.read_scene(f)
        assert inst and all(i["mesh"].startswith("/meshes/") and len(i["position"]) == 3 for i in inst), f
    (c,) = scene_file.read_scene(os.path.join(REF_SCENES, "cornell_box.ron"))
    assert c["mesh"] == "/meshes/cornell_box/scene.gltf" and np.array_equal(scene_file.instance_transform(c["position"], c["rotation"], c["scale"]),
                                                                              np.array([[2, 0, 0, 0], [0, 2, 0, -1], [0, 0, 2, 0]], np.float32))


def test_reference_cornell_scene_loads_like_the_bundled_one(emu_lib):
    """cornell_box.ron through scene_file + the glTF importer gives the geometry of kajiya_b200.scenes.cornell_box() (the bench scene):
    same depth buffer to within the 1-ulp vertex difference documented in test_asset.py"""
    import parity
    wa = World(emu_lib, 64, 64); scene_file.load_scene(wa, os.path.join(REF_SCENES, "cornell_box.ron"), REF_ASSETS); wa.set_blue_noise(scenes.blue_noise())
    scene, view = scenes.cornell_box(); wb = parity.make_world(emu_lib, scene, 64, 64)
    wa.render_frame(**view); wb.render_frame(**view)
    da, db = wa.image("depth")[..., 0], wb.image("depth")[..., 0]
    assert ((da > 0) == (db > 0)).mean() > 0.999 and np.abs(da - db).max() < 1e-5
