"""Host-side mirror of kajiya's `WorldRenderer` for the hot path (crates/lib/kajiya/src/world_renderer.rs):
add_mesh / add_instance / per-frame render, over the `kjb_world_*` C-ABI."""
import ctypes as C
import numpy as np
from ._abi import Image, Buffer, WorldDesc, WorldFrame, MeshDesc, MeshMaterial, TextureDesc, FMT_NUMPY, KjbError


def quat_from_rotation_x(angle):
    return (float(np.sin(angle / 2)), 0.0, 0.0, float(np.cos(angle / 2)))


class World:
    def __init__(self, lib, width, height, device=0, spatial_reuse_pass_count=2, enable_ircache=False, enable_rtr=False, enable_taa=False,
                 upscale=None, tile=None, use_raytraced_reservoir_visibility=False, enable_ssao=False, enable_lighting=False, hard_sun=False):
        self.lib = lib
        self.d = lib.dll
        self.ctx = C.c_void_p()
        if self.d.kjb_create(device, C.byref(self.ctx)):
            raise KjbError("kjb_create failed: " + (self.d.kjb_last_error(None) or b"").decode())
        tile_rank, tile_count = tile if tile else (0, 0)
        desc = WorldDesc(width, height, (upscale or (0, 0))[0], (upscale or (0, 0))[1], spatial_reuse_pass_count, int(use_raytraced_reservoir_visibility),
                         int(enable_ircache), int(enable_rtr), int(enable_taa), 0, 0, tile_rank, tile_count, int(enable_ssao), int(enable_lighting), int(hard_sun))
        self.w = C.c_void_p()
        if tile_count > 1 and enable_lighting:   # kjb_world_create refuses it (rc 1, no context error string: the frame driver sits above the C-ABI)
            raise KjbError("tile-sharded frames do not include the lit composite (enable_lighting): DESIGN.md §7")
        self._check(self.d.kjb_world_create(self.ctx, C.byref(desc), C.byref(self.w)))
        self.width, self.height = width, height
        self._keep = []

    def _check(self, rc):
        if rc:
            raise KjbError(f"{self.lib.backend}: rc={rc}: " + (self.d.kjb_last_error(self.ctx) or b"").decode())

    def close(self):
        if self.w:
            self.d.kjb_world_destroy(self.w); self.w = None
        if self.ctx:
            self.d.kjb_destroy(self.ctx); self.ctx = None

    def set_spatial_resolve_offsets(self, table):
        """SPATIAL_RESOLVE_OFFSETS: int32[512, 4] (rtr.rs:402-915); required when enable_rtr"""
        t = np.ascontiguousarray(table, np.int32).reshape(512, 4)
        self._check(self.d.kjb_world_set_spatial_resolve_offsets(self.w, t.ctypes.data))

    def set_debug_serial(self, on=True):
        """cache-touching passes on one device thread in launch order (deterministic; slow)"""
        self._check(self.d.kjb_set_debug_serial(self.ctx, int(on)))

    def set_option(self, option, value):
        """kjb_set_option: 1 = KJB_OPTION_HALF_RES_POSITION_CACHE (the frame driver switches it on)"""
        self._check(self.d.kjb_set_option(self.ctx, int(option), int(value)))

    # -- multi-GPU transport (tile = (rank, count)) ------------------------------------------------------------
    def comm_init_nccl(self, unique_id_bytes, rank, nranks):
        buf = C.create_string_buffer(bytes(unique_id_bytes), 128)
        self._check(self.d.kjb_comm_init_nccl(self.ctx, buf, rank, nranks))

    def comm_set_callback(self, fn, rank, nranks):
        """fn(send_ptr, recv_ptr, bytes_per_rank) -> 0; used by the CPU test builds (gloo) and custom transports"""
        CB = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64)
        self._cb = CB(lambda user, send, recv, n: int(fn(send, recv, n) or 0))
        self._check(self.d.kjb_comm_set_callback(self.ctx, C.cast(self._cb, C.c_void_p), None, rank, nranks))

    # -- scene -------------------------------------------------------------------------------------------------
    def add_mesh(self, mesh, use_lights=False):
        """mesh: dict(positions[n,3], normals[n,3], indices[m], material_ids[n], materials=[dict], uvs?, colors?)"""
        pos = np.ascontiguousarray(mesh["positions"], np.float32); nrm = np.ascontiguousarray(mesh["normals"], np.float32)
        idx = np.ascontiguousarray(mesh["indices"], np.uint32); mid = np.ascontiguousarray(mesh["material_ids"], np.uint32)
        uvs = np.ascontiguousarray(mesh["uvs"], np.float32) if mesh.get("uvs") is not None else None
        col = np.ascontiguousarray(mesh["colors"], np.float32) if mesh.get("colors") is not None else None
        mats = (MeshMaterial * len(mesh["materials"]))()
        maps = []
        texel_keep = []
        for i, m in enumerate(mesh["materials"]):
            mm = mats[i]
            mm.base_color_mult[:] = m.get("base_color", [1, 1, 1, 1])
            mm.roughness_mult = m.get("roughness", 1.0); mm.metalness_factor = m.get("metallic", 1.0)
            mm.emissive[:] = m.get("emissive", [0, 0, 0]); mm.flags = 0
            for k in range(4):
                mm.map_transforms[k * 6:(k + 1) * 6] = [1, 0, 0, 1, 0, 0]
            # load_gltf_material (kajiya-asset/src/mesh.rs:120-255): placeholders for missing maps, order normal/spec/albedo/emissive
            placeholders = [(127, 127, 255, 255), (255, 255, 127, 255), (255, 255, 255, 255), (255, 255, 255, 255)]
            for k, key in enumerate(("normal_map", "spec_map", "albedo_map", "emissive_map")):
                tex = m.get(key)
                if tex is None:
                    texels = np.array([placeholders[k]], np.uint8); w = h = mips = 1; srgb = 0
                else:
                    texels, w, h, mips, srgb = tex
                texels = np.ascontiguousarray(texels, np.uint8); texel_keep.append(texels)
                maps.append(TextureDesc(texels.ctypes.data, w, h, mips, srgb))
                mm.maps[k] = len(maps) - 1
        maps_arr = (TextureDesc * len(maps))(*maps)
        md = MeshDesc(pos.ctypes.data, nrm.ctypes.data, uvs.ctypes.data if uvs is not None else None, col.ctypes.data if col is not None else None,
                      mid.ctypes.data, idx.ctypes.data, len(pos), len(idx), mats, len(mats), maps_arr, len(maps), int(use_lights))
        h = C.c_uint32()
        self._check(self.d.kjb_world_add_mesh(self.w, C.byref(md), C.byref(h)))
        return h.value

    def add_mesh_desc(self, desc, use_lights=False):
        """add_mesh with a ready kjb_mesh_desc, e.g. `asset.GltfScene(path).desc` (the asset must outlive this call only)"""
        desc.use_lights = int(use_lights)
        h = C.c_uint32()
        self._check(self.d.kjb_world_add_mesh(self.w, C.byref(desc), C.byref(h)))
        return h.value

    def add_instance(self, mesh, transform3x4):
        t = (C.c_float * 12)(*np.asarray(transform3x4, np.float32).reshape(12))
        h = C.c_uint32()
        self._check(self.d.kjb_world_add_instance(self.w, mesh, C.byref(t), C.byref(h)))
        return h.value

    def set_instance_transform(self, handle, transform):
        t = (C.c_float * 12)(*np.asarray(transform, np.float32).reshape(-1)[:12])
        self._check(self.d.kjb_world_set_instance_transform(self.w, handle, C.byref(t)))

    def set_sun_color_multiplier(self, rgb):
        self._check(self.d.kjb_world_set_sun_color_multiplier(self.w, C.byref((C.c_float * 3)(*rgb))))

    def set_sky_ambient(self, rgb):
        self._check(self.d.kjb_world_set_sky_ambient(self.w, C.byref((C.c_float * 3)(*rgb))))

    def set_render_overrides(self, flags=0, material_roughness_scale=1.0):
        """RenderOverrides: 1 FORCE_FACE_NORMALS, 2 NO_NORMAL_MAPS, 4 FLIP_NORMAL_MAP_YZ, 8 NO_METAL; roughness scale as in the view app's GUI"""
        self._check(self.d.kjb_world_set_render_overrides(self.w, int(flags), float(material_roughness_scale)))

    def reset_reference_accumulation(self):
        self._check(self.d.kjb_world_reset_reference_accumulation(self.w))

    def set_debug_shading_mode(self, mode):
        self._check(self.d.kjb_world_set_debug_shading_mode(self.w, int(mode)))

    def set_sun_size_multiplier(self, m):
        """WorldRenderer::sun_size_multiplier: 1 = the real sun disk, 0 = point sun (skips the shadow denoiser)"""
        self._check(self.d.kjb_world_set_sun_size_multiplier(self.w, float(m)))

    def remove_instance(self, handle):
        """WorldRenderer::remove_instance (swap_remove: the last instance takes the freed slot)"""
        self._check(self.d.kjb_world_remove_instance(self.w, handle))

    def set_instance_emissive_multiplier(self, handle, value):
        self._check(self.d.kjb_world_set_instance_emissive_multiplier(self.w, handle, float(value)))

    def set_blue_noise(self, rgba8):
        a = np.ascontiguousarray(rgba8, np.uint8); assert a.size == 256 * 256 * 4
        self._check(self.d.kjb_world_set_blue_noise(self.w, a.ctypes.data))

    # -- frames ------------------------------------------------------------------------------------------------
    def _frame(self, camera_position, camera_rotation, sun_direction, vfov=52.0, host_inputs=None, host_result=None, capture_slot=0, replay_slot=0, streaming=False):
        f = WorldFrame()
        f.camera_position[:] = camera_position; f.camera_rotation[:] = camera_rotation
        f.vertical_fov_deg = vfov; f.near_plane = 0.01; f.sun_direction[:] = sun_direction; f.delta_time_seconds = 1.0 / 60.0
        if host_inputs is not None:
            f.host_gbuffer, f.host_depth, f.host_geometric_normal, f.host_velocity = host_inputs
        if host_result is not None:
            f.host_result = host_result
        f.capture_slot, f.replay_slot = capture_slot, replay_slot
        f.streaming = int(streaming)
        return f

    def render_frame(self, camera_position, camera_rotation, sun_direction, **kw):
        f = self._frame(camera_position, camera_rotation, sun_direction, **kw)
        self._check(self.d.kjb_world_render_frame(self.w, C.byref(f)))

    def render_reference(self, camera_position, camera_rotation, sun_direction, indirect_only=False, **kw):
        f = self._frame(camera_position, camera_rotation, sun_direction, **kw)
        self._check(self.d.kjb_world_render_reference(self.w, C.byref(f), int(indirect_only)))

    def wait(self):
        """block until every streaming frame has delivered its host_result"""
        self._check(self.d.kjb_world_wait(self.w))

    def sync(self):
        self._check(self.d.kjb_sync(self.ctx))

    def set_profiling(self, on):
        self.d.kjb_world_set_profiling(self.w, int(on))

    def pass_timings(self):
        """{label: (calls, total_ms)} of the passes run since profiling was switched on"""
        out = {}
        for line in self.d.kjb_world_pass_timings(self.w).decode().split("\n"):
            if line:
                label, calls, ms = line.split("\t"); out[label] = (int(calls), float(ms))
        return out

    def timer_record(self, slot):
        self._check(self.d.kjb_timer_record(self.ctx, slot))

    def timer_elapsed_ms(self, a, b):
        ms = C.c_float()
        self._check(self.d.kjb_timer_elapsed_ms(self.ctx, a, b, C.byref(ms)))
        return ms.value

    def stop_after(self, label):
        self.d.kjb_world_set_stop_after(self.w, (label or "").encode())

    def result_rows(self):
        """(y0, y1): the rows of the result image (the TAA output, else the render-res result) this world renders and writes into host_result —
        a tile-sharded world's band on the result grid, the whole image otherwise (kjb_world_result_rows)"""
        y0, y1 = C.c_uint32(), C.c_uint32()
        self._check(self.d.kjb_world_result_rows(self.w, C.byref(y0), C.byref(y1)))
        return y0.value, y1.value

    def device_read(self, ptr, nbytes):
        """bytes of the context's memory at `ptr` (device memory on the CUDA build), e.g. the send buffer handed to a host all-gather callback"""
        out = np.empty(int(nbytes), np.uint8)
        self._check(self.d.kjb_buffer_download(self.ctx, C.byref(Buffer(ptr, nbytes)), 0, out.ctypes.data, nbytes))
        return out

    def device_write(self, ptr, host):
        """copy the contiguous array `host` to the context's memory at `ptr` (the receive buffer of a host all-gather callback)"""
        a = np.ascontiguousarray(host)
        self._check(self.d.kjb_buffer_upload(self.ctx, C.byref(Buffer(ptr, a.nbytes)), 0, a.ctypes.data, a.nbytes))
        self.sync()

    @property
    def frame_index(self):
        return self.d.kjb_world_frame_index(self.w)

    def stats(self):
        s = (C.c_uint64 * 4)()
        self.d.kjb_world_last_frame_stats(self.w, C.byref(s))
        return dict(launches=s[0], closest_rays=s[1], any_hit_rays=s[2], passes=s[3])

    def set_cuda_graph(self, on):
        """one CUDA graph launch per frame instead of ~40 kernel launches (default on; applies from the fifth frame)"""
        self._check(self.d.kjb_world_set_cuda_graph(self.w, int(on)))

    def set_async_compute(self, on):
        """irradiance-cache chain on the async pass queue, under the previous frame's reflection filters + TAA (default on; CUDA backend)"""
        self._check(self.d.kjb_world_set_async_compute(self.w, int(on)))

    def graph_stats(self):
        s = (C.c_uint64 * 2)()
        self._check(self.d.kjb_graph_stats(self.ctx, C.byref(s)))
        return dict(launches=s[0], instantiations=s[1])

    def tlas_stats(self):
        """how "rebuild tlas" was served: full rebuilds vs device refits (transform-only changes)"""
        s = (C.c_uint64 * 2)()
        self._check(self.d.kjb_tlas_stats(self.ctx, C.byref(s)))
        return dict(rebuilds=s[0], refits=s[1])

    def tlas_download(self):
        """the acceleration structure as built (include/kjb_tlas.h): dict of raw arrays — nodes uint32[n, 16] (64-byte nodes), tris
        uint32[slots, 12] (48-byte leaf-order records, global id in word 3), tri_info uint32[triangles, 2] (instance, primitive), parent
        int32[n] — and root (a node index, or a leaf / empty reference)"""
        if not self.lib.has_tlas_download:
            raise KjbError(f"{self.lib.backend} does not expose its acceleration structure")
        counts, root = (C.c_uint32 * 3)(), C.c_int32()
        self._check(self.d.kjb_tlas_download(self.ctx, C.byref(counts), C.byref(root), None, None, None, None))
        nodes, tris = np.zeros((counts[0], 16), np.uint32), np.zeros((counts[1], 12), np.uint32)
        info, parent = np.zeros((counts[2], 2), np.uint32), np.zeros(counts[0], np.int32)
        self._check(self.d.kjb_tlas_download(self.ctx, C.byref(counts), C.byref(root), nodes.ctypes.data, tris.ctypes.data, info.ctypes.data, parent.ctypes.data))
        return dict(nodes=nodes, tris=tris, tri_info=info, parent=parent, root=int(root.value))

    def trace_rays(self, rays, any_hit=False, cull_back=False, brute_force=False):
        """rays float32[n, 8] (o.xyz, tmin, d.xyz, tmax) against the structure as built (include/kjb_tlas.h: kjb_tlas_trace) -> uint32[n, 4]:
        t, u, v as float bits and the global triangle id, (0, 0, 0, 0xffffffff) for a miss; with any_hit only column 3 counts (0 = hit).
        brute_force tests every triangle record instead of walking the tree."""
        if not self.lib.has_tlas_trace:
            raise KjbError(f"{self.lib.backend} does not expose its acceleration structure")
        r = np.ascontiguousarray(rays, np.float32).reshape(-1, 8)
        out = np.zeros((len(r), 4), np.uint32)
        flags = (1 if any_hit else 0) | (2 if cull_back else 0) | (4 if brute_force else 0)   # KJB_TLAS_TRACE_*
        self._check(self.d.kjb_tlas_trace(self.ctx, r.ctypes.data, len(r), flags, out.ctypes.data))
        return out

    # -- images ------------------------------------------------------------------------------------------------
    def image_names(self):
        return [n for n in self.d.kjb_world_image_names(self.w).decode().split("\n") if n]

    def image_handle(self, name):
        img = Image()
        if self.d.kjb_world_get_image(self.w, name.encode(), C.byref(img)):
            raise KeyError(name)
        return img

    def image(self, name):
        """Download an image as a numpy array [layers*height, width, components] of its storage dtype."""
        img = self.image_handle(name)
        dt, comps = FMT_NUMPY[img.format]
        out = np.empty((img.layers * img.height, img.width, comps), dt)
        self._check(self.d.kjb_image_download(self.ctx, C.byref(img), out.ctypes.data))
        self.sync()
        return out
