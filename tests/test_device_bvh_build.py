"""The acceleration structure built on the device ("rebuild tlas" when the instance list changes, kajiya_b200/csrc/kjb_bvh_build.cuh) is the
tree of the host binned-SAH builder (kajiya_b200/csrc/kjb_bvh.cpp): nodes and parent links byte for byte, tri_info identical, the same triangles
in every leaf (ascending global id on the device).  Where the host's split depended on its list order the device halves the gid-ordered
segment: such trees stay well-formed and render the same frames.  The build does not depend on the launch order, a dynamic scene renders
bit for bit like the oracle after every frame, and on the GPU a rebuild runs inside a CUDA-graph recording."""
import ctypes as C
import numpy as np
import pytest
import conftest
import parity
from kajiya_b200 import scenes, asset
from kajiya_b200.world import World

ORDERS = ((0, 0), (1, 0), (2, 1), (2, 0x9E3779B9))   # kjb_emu_set_launch_order: forward, reverse, two permutations
ORDERED_CACHE_SCHEDULE = 2


# ------------------------------------------------------------------------------------------------ helpers
world_triangles = parity.world_triangles


def reference_tree(world_tris):
    """the host builder over the same triangles (exported by the emulator library)"""
    d = C.CDLL(conftest.EMU_SO)
    d.kjb_ref_bvh_build.restype = C.c_void_p; d.kjb_ref_bvh_build.argtypes = [C.c_void_p, C.c_uint32]
    d.kjb_ref_bvh_counts.argtypes = [C.c_void_p, C.POINTER(C.c_uint32 * 2), C.POINTER(C.c_int32)]
    d.kjb_ref_bvh_copy.argtypes = [C.c_void_p] * 4
    d.kjb_ref_bvh_free.argtypes = [C.c_void_p]
    wt = np.ascontiguousarray(world_tris, np.float32)
    h = d.kjb_ref_bvh_build(wt.ctypes.data, len(wt))
    try:
        counts, root = (C.c_uint32 * 2)(), C.c_int32()
        d.kjb_ref_bvh_counts(h, C.byref(counts), C.byref(root))
        nodes, tris, parent = np.zeros((counts[0], 16), np.uint32), np.zeros((counts[1], 12), np.uint32), np.zeros(counts[0], np.int32)
        d.kjb_ref_bvh_copy(h, nodes.ctypes.data, tris.ctypes.data, parent.ctypes.data)
    finally:
        d.kjb_ref_bvh_free(h)
    return dict(nodes=nodes, tris=tris, parent=parent, root=int(root.value))


def leaves(tree):
    """(first, count) of every leaf, from the root reference and the child references"""
    refs = [tree["root"]] if tree["root"] < 0 else list(tree["nodes"][:, 12:14].view(np.int32).ravel())
    out = []
    for r in refs:
        if r < 0 and r != -1:
            e = ~int(r)
            out.append((e >> 3, (e & 7) + 1))
    if tree["root"] == -1 and not len(tree["nodes"]):
        return []
    return sorted(out)


def sorted_in_leaves(tree):
    """the triangle records with every leaf's records in ascending global id"""
    t = tree["tris"].copy()
    for first, count in leaves(tree):
        seg = t[first:first + count]
        t[first:first + count] = seg[np.argsort(seg[:, 3], kind="stable")]
    return t


def assert_same_tree(dev, ref, info):
    assert dev["root"] == ref["root"]
    assert dev["nodes"].shape == ref["nodes"].shape and dev["nodes"].tobytes() == ref["nodes"].tobytes()
    assert np.array_equal(dev["parent"], ref["parent"])
    assert np.array_equal(dev["tri_info"], info)
    assert dev["tris"].shape == ref["tris"].shape
    assert np.array_equal(sorted_in_leaves(dev), sorted_in_leaves(ref))
    for first, count in leaves(dev):   # the device keeps ascending global id inside a leaf
        assert (np.diff(dev["tris"][first:first + count, 3].astype(np.int64)) > 0).all()


def built_tree(lib, scene, **kw):
    """a world over `scene`, one tiny frame (which runs "rebuild tlas"), and its structure"""
    w = parity.make_world(lib, scene, 16, 8, **kw)
    _, view = scenes.cornell_box()
    w.render_frame(**view)
    return w, w.tlas_download()


def check_well_formed(tree, world_tris):
    """every triangle in exactly one leaf, every slot box contains what is below it, depth within the traversal stack (64)"""
    nodes = tree["nodes"]; n = len(world_tris)
    box = nodes[:, :12].view(np.float32)
    slot_lo = lambda i, k: np.array([box[i, 4 * k], box[i, 4 * k + 2], box[i, 8 + 2 * k]])
    slot_hi = lambda i, k: np.array([box[i, 4 * k + 1], box[i, 4 * k + 3], box[i, 8 + 2 * k + 1]])
    gids = np.concatenate([tree["tris"][f:f + c, 3] for f, c in leaves(tree)])
    assert np.array_equal(np.sort(gids), np.arange(n))
    v = world_tris.reshape(-1, 3, 3)
    tlo, thi = v.min(1), v.max(1)
    stack, max_depth = [(0, 1)], 0
    while stack:
        i, d = stack.pop()
        max_depth = max(max_depth, d)
        for k in range(2):
            ch = int(nodes[i, 12 + k].view(np.int32))
            lo, hi = slot_lo(i, k), slot_hi(i, k)
            if ch >= 0:
                for kk in range(2):
                    assert (lo <= slot_lo(ch, kk)).all() and (slot_hi(ch, kk) <= hi).all()
                assert tree["parent"][ch] == (i << 1) | k
                stack.append((ch, d + 1))
            else:
                e = ~ch; g = tree["tris"][e >> 3:(e >> 3) + (e & 7) + 1, 3]
                assert (lo <= tlo[g]).all() and (thi[g] <= hi).all()
    assert max_depth <= 64
    return max_depth


def tiny_mesh(n_tris, x0=0.0):
    p = np.array([[x0 + 0.1 * i, 0.2, 0.1 * (i % 2)] for i in range(n_tris + 2)], np.float32)
    idx = np.array([[i, i + 1, i + 2] for i in range(n_tris)], np.uint32).ravel()
    return dict(positions=p, normals=np.tile(np.array([[0, 0, 1]], np.float32), (len(p), 1)), indices=idx,
                material_ids=np.zeros(len(p), np.uint32), materials=[dict(base_color=[0.8, 0.7, 0.6, 1.0], roughness=0.5)])


def exponential_strip(n=200):
    """triangles spaced exponentially along x, below the Cornell floor: the SAH splits peel a few triangles off at a time (depth 31)"""
    p, idx = [], []
    for i in range(n):
        x = float(1.5 ** i) * 0.01
        b = len(p)
        p += [[x, -3.0, 0.0], [x + 0.001, -3.0, 0.0], [x, -3.0, 0.001]]
        idx += [b, b + 1, b + 2]
    p = np.array(p, np.float32)
    return dict(positions=p, normals=np.tile(np.array([[0, 1, 0]], np.float32), (len(p), 1)), indices=np.array(idx, np.uint32),
                material_ids=np.zeros(len(p), np.uint32), materials=[dict(base_color=[0.5, 0.5, 0.5, 1.0], roughness=0.8)])


def _rot_y(a, s=1.0, t=(0.0, 0.0, 0.0)):
    c, n = np.cos(a) * s, np.sin(a) * s
    return np.array([[c, 0, n, t[0]], [0, s, 0, t[1]], [-n, 0, c, t[2]]], np.float32)


def _courtyard():
    path = conftest.os.path.join(conftest.ROOT, "tests", "golden", "gltf", "courtyard.gltf")
    a = asset.GltfScene(path).arrays()
    mesh = dict(positions=a["positions"], normals=a["normals"], indices=a["indices"], material_ids=np.zeros(len(a["positions"]), np.uint32),
                materials=[dict(base_color=[0.7, 0.7, 0.7, 1.0], roughness=0.6)])
    return [(mesh, [np.eye(3, 4, dtype=np.float32)])]


def _scene(name):
    cornell, _ = scenes.cornell_box()
    mesh, transforms = cornell[0]
    if name == "cornell":
        return cornell
    if name == "cornell_x2":
        return [(mesh, [transforms[0], _rot_y(0.6, 0.4, (0.3, 0.1, -0.2))])]
    if name == "cornell_x3":
        return [(mesh, [transforms[0], _rot_y(0.6, 0.4, (0.3, 0.1, -0.2)), _rot_y(-1.1, 0.25, (-0.4, 0.5, 0.3))])]
    if name == "atrium_20k":
        return scenes.atrium(target_tris=20000)[0]
    if name == "courtyard":
        return _courtyard()
    if name == "four_triangles":
        return [(tiny_mesh(4), [np.eye(3, 4, dtype=np.float32)])]
    if name == "no_instances":
        return []
    raise KeyError(name)


# ------------------------------------------------------------------------------------------------ CPU (emulator)
@pytest.mark.parametrize("name", ["cornell", "cornell_x2", "cornell_x3", "atrium_20k", "courtyard", "four_triangles", "no_instances"])
def test_device_tree_equals_the_host_reference(emu_lib, name):
    scene = _scene(name)
    wt, info = world_triangles(scene)
    w, dev = built_tree(emu_lib, scene)
    assert_same_tree(dev, reference_tree(wt), info)
    if name == "four_triangles":
        assert dev["root"] == ~3 and len(dev["nodes"]) == 0
    if name == "no_instances":
        assert dev["root"] == -1 and len(dev["tris"]) == 1 and not dev["tris"].any()
    assert w.tlas_stats() == dict(rebuilds=1, refits=0)


@pytest.mark.parametrize("case", ["coincident_centroids", "deep_strip"])
def test_order_dependent_fallbacks_stay_well_formed(oracle_lib, emu_lib, case):
    cornell, view = scenes.cornell_box()
    mesh, transforms = cornell[0]
    if case == "coincident_centroids":
        scene = [(mesh, [transforms[0]] * 6)]                  # every triangle six times: segments of identical centroids, split by halving
    else:
        scene = [(mesh, [transforms[0]]), (exponential_strip(), [np.eye(3, 4, dtype=np.float32)])]
    wt, _ = world_triangles(scene)
    we = parity.make_world(emu_lib, scene, 48, 32, enable_rtr=True, enable_taa=True)
    wo = parity.make_world(oracle_lib, scene, 48, 32, enable_rtr=True, enable_taa=True)
    for f in range(2):
        we.render_frame(**view); wo.render_frame(**view)
        bad = parity.compare_images(wo, we)
        assert not bad, (f, bad[:8])
    tree = we.tlas_download()
    depth = check_well_formed(tree, wt)
    if case == "deep_strip":
        assert depth >= 30
    else:   # the fallback ran: some node over 5 or 6 copies of one triangle, split into two leaves
        cent = lambda g: (wt[g].reshape(-1, 3, 3).min(1) + wt[g].reshape(-1, 3, 3).max(1)) * np.float32(0.5)
        halved = 0
        for i in range(len(tree["nodes"])):
            ch = tree["nodes"][i, 12:14].view(np.int32)
            if (ch < 0).all():
                g = np.concatenate([tree["tris"][(~int(c)) >> 3:((~int(c)) >> 3) + ((~int(c)) & 7) + 1, 3] for c in ch])
                halved += len(g) > 4 and (cent(g) == cent(g)[0]).all()
        assert halved > 0


def test_build_does_not_depend_on_the_launch_order(emu_lib):
    f = emu_lib.dll.kjb_emu_set_launch_order
    f.argtypes, f.restype = [C.c_int, C.c_uint32], None
    scene = _scene("atrium_20k")
    got = {}
    try:
        for mode, seed in ORDERS:
            f(mode, seed)
            _, t = built_tree(emu_lib, scene)
            got[(mode, seed)] = b"".join(t[k].tobytes() for k in ("nodes", "tris", "tri_info", "parent"))
    finally:
        f(0, 0)
    assert len(set(got.values())) == 1


def _dynamic_sequence(worlds, view, check):
    """add an instance, move it (a refit of a device-built tree), remove another (swap_remove), add another mesh, remove down to one;
    check(frame) after every frame.  Returns the (rebuilds, refits) "rebuild tlas" must have served."""
    cornell, _ = scenes.cornell_box()
    mesh, transforms = cornell[0]
    small = lambda dx: np.array([[0.25, 0, 0, 0.1 + dx], [0, 0.25, 0, 0.3], [0, 0, 0.25, 0.2]], np.float32)
    st = []
    for w in worlds:
        hm, ht = w.add_mesh(mesh), w.add_mesh(tiny_mesh(6, -0.5))
        st.append(dict(hm=hm, ht=ht, base=[w.add_instance(hm, transforms[0]), w.add_instance(hm, small(-0.4))]))
        w.set_blue_noise(scenes.blue_noise()); w.set_spatial_resolve_offsets(scenes.spatial_resolve_offsets())
    steps = [("first", "rebuild"), ("add", "rebuild"), ("move", "refit"), ("move", "refit"), ("remove_other", "rebuild"), ("add_mesh", "rebuild"),
             ("still", None), ("remove_mesh", "rebuild"), ("remove_added", "rebuild")]
    for f, (step, _) in enumerate(steps):
        for w, s in zip(worlds, st):
            if step == "add":
                s["new"] = w.add_instance(s["hm"], small(0.0))
            elif step == "move":
                s["dx"] = s.get("dx", 0.0) + 0.05
                w.set_instance_transform(s["new"], small(s["dx"]))
            elif step == "remove_other":
                w.remove_instance(s["base"][1])          # swap_remove: the added instance takes its slot
            elif step == "add_mesh":
                s["tiny"] = w.add_instance(s["ht"], np.eye(3, 4, dtype=np.float32))
            elif step == "remove_mesh":
                w.remove_instance(s["tiny"])
            elif step == "remove_added":
                w.remove_instance(s["new"])              # one instance left
            w.render_frame(**view)
        check(f)
    return sum(k == "rebuild" for _, k in steps), sum(k == "refit" for _, k in steps)


def test_dynamic_scene_matches_the_oracle_every_frame(oracle_lib, emu_lib):
    _, view = scenes.cornell_box()
    kw = dict(enable_rtr=True, enable_taa=True)
    wo, we = World(oracle_lib, 64, 40, **kw), World(emu_lib, 64, 40, **kw)

    def check(f):
        bad = parity.compare_images(wo, we)
        assert not bad, (f, bad[:8])
    rebuilds, refits = _dynamic_sequence([wo, we], view, check)
    assert we.tlas_stats() == dict(rebuilds=rebuilds, refits=refits)
    assert (rebuilds, refits) == (6, 2)


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["atrium", "ruins"])
def test_gpu_device_tree_equals_the_host_reference(cuda_lib, name):
    scene = scenes.atrium()[0] if name == "atrium" else scenes.ruins()[0]
    wt, info = world_triangles(scene)
    _, dev = built_tree(cuda_lib, scene)
    assert_same_tree(dev, reference_tree(wt), info)


@pytest.mark.gpu
def test_gpu_dynamic_scene_matches_the_emulator_every_frame(cuda_lib, emu_lib):
    """the full path (rtdgi, irradiance cache, reflections, TAA) on the atrium's 480x270 frame, CUDA graphs and the async cache chain on (the
    defaults): every image and cache buffer bit for bit against the emulator on the ordered cache schedule, through the dynamic sequence"""
    scene, view = scenes.atrium()
    kw = dict(enable_ircache=True, enable_rtr=True, enable_taa=True, spatial_reuse_pass_count=2)
    wg, we = World(cuda_lib, 480, 270, **kw), World(emu_lib, 480, 270, **kw)
    we.set_option(ORDERED_CACHE_SCHEDULE, 1)
    for w in (wg, we):
        for mesh, transforms in scene:
            h = w.add_mesh(mesh)
            for t in transforms:
                w.add_instance(h, t)

    def check(f):
        bad = parity.compare_images(wg, we)
        assert not bad, (f, bad[:8])
    rebuilds, refits = _dynamic_sequence([wg, we], view, check)
    assert wg.tlas_stats() == dict(rebuilds=rebuilds, refits=refits) == we.tlas_stats()
    assert wg.graph_stats()["launches"] > 0


class _Instance(C.Structure):   # kjb_instance (kjb.h)
    _fields_ = [("transform", C.c_float * 12), ("mesh_index", C.c_uint32), ("emissive_multiplier", C.c_float)]


@pytest.mark.gpu
def test_gpu_rebuild_inside_a_graph_recording(cuda_lib):
    """with capacities reserved, a rebuild that changes the instance list neither synchronises nor allocates: it is recorded into a CUDA graph
    (relaxed capture is invalidated by any synchronising call) and the frames after it equal those of a world that rebuilt directly"""
    d = cuda_lib.dll
    d.kjb_rebuild_tlas.argtypes, d.kjb_rebuild_tlas.restype = [C.c_void_p, C.c_void_p, C.c_uint32], C.c_int
    d.kjb_graph_begin.argtypes = d.kjb_graph_end.argtypes = [C.c_void_p]
    d.kjb_graph_begin.restype = d.kjb_graph_end.restype = C.c_int
    cornell, view = scenes.cornell_box()
    mesh, transforms = cornell[0]
    extra = [transforms[0], _rot_y(0.6, 0.4, (0.3, 0.1, -0.2)), _rot_y(-1.1, 0.25, (-0.4, 0.5, 0.3))]
    worlds = [parity.make_world(cuda_lib, [(mesh, extra)], 160, 90, enable_rtr=True, enable_taa=True) for _ in range(2)]
    for f in range(5):
        for w in worlds:
            w.render_frame(**view)
    for w in worlds:
        w.remove_instance(1)                  # handles 0, 1, 2 in add order: swap_remove leaves (0, 2)
    kept = [extra[0], extra[2]]
    arr = (_Instance * 2)()
    for i, t in enumerate(kept):
        arr[i].transform[:] = list(np.asarray(t, np.float32).reshape(12)); arr[i].mesh_index = 0; arr[i].emissive_multiplier = 1.0
    wg = worlds[0]
    before = wg.tlas_stats()
    assert d.kjb_graph_begin(wg.ctx) == 0
    rc = d.kjb_rebuild_tlas(wg.ctx, C.cast(arr, C.c_void_p), 2)
    end = d.kjb_graph_end(wg.ctx)
    assert rc == 0 and end == 0, (d.kjb_last_error(wg.ctx) or b"").decode()
    assert wg.tlas_stats()["rebuilds"] == before["rebuilds"] + 1
    for f in range(3):
        for w in worlds:
            w.render_frame(**view)
        bad = parity.compare_images(worlds[0], worlds[1])
        assert not bad, (f, bad[:8])
    assert wg.tlas_stats() == worlds[1].tlas_stats()   # the world's own rebuild found the list unchanged
    wt, info = world_triangles([(mesh, kept)])
    assert_same_tree(wg.tlas_download(), reference_tree(wt), info)
