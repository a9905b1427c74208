"""GPU twins of features whose CPU-emulator versions are in test_emu_parity.py / test_multigpu_gloo.py (bit-exact against the oracle).
The file sorts last on purpose: a `pytest -m gpu` run reaches it after every older GPU test."""
import os
import numpy as np, pytest
import conftest, parity
from kajiya_b200 import scenes


@pytest.mark.gpu
def test_everything_at_once_on_gpu(oracle_lib, cuda_lib):
    """the all-features configuration of test_emu_parity.py::test_everything_at_once (incl. LightingRenderer::render_specular, which has
    no other GPU coverage) with the racy cache passes on the deterministic serial schedule: every image bit for bit"""
    from kajiya_b200 import asset
    from kajiya_b200.world import World
    path = os.path.join(conftest.ROOT, "tests", "golden", "gltf", "courtyard.gltf")
    view = dict(camera_position=(0.5, 2.5, 7.0), camera_rotation=(float(np.sin(-0.15)), 0.0, 0.0, float(np.cos(-0.15))), sun_direction=(0.35, 0.8, 0.45))
    kw = dict(spatial_reuse_pass_count=2, use_raytraced_reservoir_visibility=True, enable_ircache=True, enable_rtr=True, enable_ssao=True, enable_lighting=True, enable_taa=True, upscale=(108, 72))
    worlds = []
    for lib in (oracle_lib, cuda_lib):
        sc = asset.GltfScene(path)
        w = World(lib, 72, 48, **kw)
        w.add_instance(w.add_mesh_desc(sc.desc, use_lights=True), np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]], np.float32))
        w.set_blue_noise(scenes.blue_noise()); w.set_spatial_resolve_offsets(scenes.spatial_resolve_offsets())
        sc.close(); worlds.append(w)
    wa, wb = worlds
    wb.set_debug_serial(True)
    for f in range(4):
        v = dict(view); px, py, pz = view["camera_position"]
        v["camera_position"] = (px + 0.25 * np.sin(0.7 * f), py + 0.05 * f, pz - 0.1 * f)
        wa.render_frame(**v); wb.render_frame(**v)
        assert not parity.compare_images(wa, wb), f
    assert "lighting.refl0" in wb.image_names()
