"""ctypes binding of the C-ABI declared in include/kjb.h and include/kjb_world.h.

`KjbLib(path)` binds one shared library that exports the ABI.  The product only ever binds
kajiya_b200/csrc/libkjb.so (the CUDA build); the test-suite binds the oracle and the CPU kernel
emulator through the same class, which is what makes the parity tests symmetrical.
"""
import ctypes as C
import numpy as np

# kjb_format
FMT = dict(R32_FLOAT=1, RG32_UINT=2, RGBA32_FLOAT=3, RGBA32_UINT=4, RGBA16_FLOAT=5, RG16_FLOAT=6, RGBA8_UNORM=7,
           RGBA8_SNORM=8, R8_UNORM=9, R8_SNORM=10, RGBA16_SNORM=11, A2R10G10B10_UNORM=12, R11G11B10_UFLOAT=13,
           R32_UINT=14, R16_FLOAT=15, RG32_FLOAT=16)
FMT_NAME = {v: k for k, v in FMT.items()}
# numpy view of one texel of each format: (dtype, components)
FMT_NUMPY = {1: (np.float32, 1), 2: (np.uint32, 2), 3: (np.float32, 4), 4: (np.uint32, 4), 5: (np.float16, 4), 6: (np.float16, 2),
             7: (np.uint8, 4), 8: (np.int8, 4), 9: (np.uint8, 1), 10: (np.int8, 1), 11: (np.int16, 4), 12: (np.uint32, 1),
             13: (np.uint32, 1), 14: (np.uint32, 1), 15: (np.float16, 1), 16: (np.float32, 2)}


class Image(C.Structure):
    _fields_ = [("data", C.c_void_p), ("width", C.c_uint32), ("height", C.c_uint32), ("format", C.c_uint32), ("layers", C.c_uint32)]


class Buffer(C.Structure):
    _fields_ = [("data", C.c_void_p), ("size_bytes", C.c_uint64)]


class MeshMaterial(C.Structure):   # kjb_mesh_material, 152 bytes
    _fields_ = [("base_color_mult", C.c_float * 4), ("maps", C.c_uint32 * 4), ("roughness_mult", C.c_float), ("metalness_factor", C.c_float),
                ("emissive", C.c_float * 3), ("flags", C.c_uint32), ("map_transforms", C.c_float * 24)]


class TextureDesc(C.Structure):
    _fields_ = [("texels", C.c_void_p), ("width", C.c_uint32), ("height", C.c_uint32), ("mip_count", C.c_uint32), ("srgb", C.c_uint32)]


class WorldDesc(C.Structure):
    _fields_ = [("render_width", C.c_uint32), ("render_height", C.c_uint32), ("temporal_upscale_width", C.c_uint32), ("temporal_upscale_height", C.c_uint32),
                ("spatial_reuse_pass_count", C.c_uint32), ("use_raytraced_reservoir_visibility", C.c_uint32),
                ("enable_ircache", C.c_uint32), ("enable_rtr", C.c_uint32), ("enable_taa", C.c_uint32), ("tile_y0", C.c_uint32), ("tile_y1", C.c_uint32),
                ("tile_rank", C.c_uint32), ("tile_count", C.c_uint32), ("enable_ssao", C.c_uint32), ("enable_lighting", C.c_uint32), ("hard_sun", C.c_uint32)]


class MeshDesc(C.Structure):
    _fields_ = [("positions", C.c_void_p), ("normals", C.c_void_p), ("uvs", C.c_void_p), ("colors", C.c_void_p), ("material_ids", C.c_void_p),
                ("indices", C.c_void_p), ("vertex_count", C.c_uint32), ("index_count", C.c_uint32), ("materials", C.POINTER(MeshMaterial)),
                ("material_count", C.c_uint32), ("maps", C.POINTER(TextureDesc)), ("map_count", C.c_uint32), ("use_lights", C.c_uint32)]


class WorldFrame(C.Structure):
    _fields_ = [("camera_position", C.c_float * 3), ("camera_rotation", C.c_float * 4), ("vertical_fov_deg", C.c_float), ("near_plane", C.c_float),
                ("sun_direction", C.c_float * 3), ("delta_time_seconds", C.c_float),
                ("host_gbuffer", C.c_void_p), ("host_depth", C.c_void_p), ("host_geometric_normal", C.c_void_p), ("host_velocity", C.c_void_p),
                ("host_result", C.c_void_p), ("capture_slot", C.c_uint32), ("replay_slot", C.c_uint32), ("streaming", C.c_uint32)]


assert C.sizeof(MeshMaterial) == 152


class KjbError(RuntimeError):
    pass


class KjbLib:
    """One loaded implementation of the ABI (CUDA / emulator / oracle)."""

    def __init__(self, path):
        self.path = path
        self.dll = C.CDLL(path, mode=C.RTLD_LOCAL)
        d = self.dll
        P = C.c_void_p
        sig = {
            "kjb_abi_version": (C.c_int, []),
            "kjb_backend_name": (C.c_char_p, []),
            "kjb_create": (C.c_int, [C.c_int, C.POINTER(P)]),
            "kjb_destroy": (None, [P]),
            "kjb_sync": (C.c_int, [P]),
            "kjb_last_error": (C.c_char_p, [P]),
            "kjb_launch_count": (C.c_uint64, [P]),
            "kjb_stream": (P, [P]),
            "kjb_format_texel_bytes": (C.c_uint32, [C.c_uint32]),
            "kjb_image_alloc": (C.c_int, [P, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(Image)]),
            "kjb_image_free": (C.c_int, [P, C.POINTER(Image)]),
            "kjb_image_clear": (C.c_int, [P, C.POINTER(Image)]),
            "kjb_image_upload": (C.c_int, [P, C.POINTER(Image), P]),
            "kjb_image_download": (C.c_int, [P, C.POINTER(Image), P]),
            "kjb_ray_counters": (C.c_int, [P, C.POINTER(C.c_uint64 * 2), C.c_int]),
            "kjb_world_create": (C.c_int, [P, C.POINTER(WorldDesc), C.POINTER(P)]),
            "kjb_world_destroy": (None, [P]),
            "kjb_world_add_mesh": (C.c_int, [P, C.POINTER(MeshDesc), C.POINTER(C.c_uint32)]),
            "kjb_world_add_instance": (C.c_int, [P, C.c_uint32, C.POINTER(C.c_float * 12), C.POINTER(C.c_uint32)]),
            "kjb_world_set_instance_transform": (C.c_int, [P, C.c_uint32, C.POINTER(C.c_float * 12)]),
            "kjb_world_remove_instance": (C.c_int, [P, C.c_uint32]),
            "kjb_world_set_sun_size_multiplier": (C.c_int, [P, C.c_float]),
            "kjb_world_set_sun_color_multiplier": (C.c_int, [P, C.POINTER(C.c_float * 3)]),
            "kjb_world_set_sky_ambient": (C.c_int, [P, C.POINTER(C.c_float * 3)]),
            "kjb_world_set_render_overrides": (C.c_int, [P, C.c_uint32, C.c_float]),
            "kjb_world_set_debug_shading_mode": (C.c_int, [P, C.c_uint32]),
            "kjb_world_reset_reference_accumulation": (C.c_int, [P]),
            "kjb_world_set_instance_emissive_multiplier": (C.c_int, [P, C.c_uint32, C.c_float]),
            "kjb_world_set_blue_noise": (C.c_int, [P, P]),
            "kjb_world_set_spatial_resolve_offsets": (C.c_int, [P, P]),
            "kjb_world_render_frame": (C.c_int, [P, C.POINTER(WorldFrame)]),
            "kjb_world_render_reference": (C.c_int, [P, C.POINTER(WorldFrame), C.c_uint32]),
            "kjb_world_frame_index": (C.c_uint32, [P]),
            "kjb_world_result_rows": (C.c_int, [P, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]),
            "kjb_buffer_upload": (C.c_int, [P, C.POINTER(Buffer), C.c_uint64, P, C.c_uint64]),
            "kjb_buffer_download": (C.c_int, [P, C.POINTER(Buffer), C.c_uint64, P, C.c_uint64]),
            "kjb_world_wait": (C.c_int, [P]),
            "kjb_world_get_image": (C.c_int, [P, C.c_char_p, C.POINTER(Image)]),
            "kjb_world_image_names": (C.c_char_p, [P]),
            "kjb_world_last_frame_stats": (C.c_int, [P, C.POINTER(C.c_uint64 * 4)]),
            "kjb_world_set_stop_after": (C.c_int, [P, C.c_char_p]),
            "kjb_world_set_profiling": (C.c_int, [P, C.c_uint32]),
            "kjb_comm_nccl_unique_id": (C.c_int, [P]),
            "kjb_comm_init_nccl": (C.c_int, [P, P, C.c_uint32, C.c_uint32]),
            "kjb_comm_set_callback": (C.c_int, [P, P, P, C.c_uint32, C.c_uint32]),
            "kjb_world_pass_timings": (C.c_char_p, [P]),
            "kjb_set_debug_serial": (C.c_int, [P, C.c_uint32]),
            "kjb_tlas_stats": (C.c_int, [P, C.POINTER(C.c_uint64 * 2)]),
            "kjb_graph_stats": (C.c_int, [P, C.POINTER(C.c_uint64 * 2)]),
            "kjb_graph_select": (C.c_int, [P, C.c_uint32]), "kjb_set_pass_queue": (C.c_int, [P, C.c_uint32]), "kjb_async_passes_supported": (C.c_int, [P]),
            "kjb_world_set_cuda_graph": (C.c_int, [P, C.c_uint32]), "kjb_world_set_async_compute": (C.c_int, [P, C.c_uint32]),
            "kjb_set_option": (C.c_int, [P, C.c_uint32, C.c_uint32]),
            "kjb_timer_record": (C.c_int, [P, C.c_uint32]),
            "kjb_timer_elapsed_ms": (C.c_int, [P, C.c_uint32, C.c_uint32, C.POINTER(C.c_float)]),
        }
        self.missing = []
        for name, (res, args) in sig.items():
            try:
                fn = getattr(d, name)
            except AttributeError:
                self.missing.append(name)
                continue
            fn.restype = res
            fn.argtypes = args
        if self.missing:
            raise KjbError(f"{path} does not export: {self.missing}")
        if d.kjb_abi_version() != 1:
            raise KjbError("ABI version mismatch")
        # include/kjb_tlas.h: the CUDA library and its emulator build inspect their acceleration structure; the oracle keeps its own
        self.has_tlas_download = hasattr(d, "kjb_tlas_download")
        if self.has_tlas_download:
            d.kjb_tlas_download.restype = C.c_int
            d.kjb_tlas_download.argtypes = [P, C.POINTER(C.c_uint32 * 3), C.POINTER(C.c_int32), P, P, P, P]
        self.has_tlas_trace = hasattr(d, "kjb_tlas_trace")
        if self.has_tlas_trace:
            d.kjb_tlas_trace.restype = C.c_int
            d.kjb_tlas_trace.argtypes = [P, P, C.c_uint32, C.c_uint32, P]

    @property
    def backend(self):
        return self.dll.kjb_backend_name().decode()


# every symbol include/kjb.h + include/kjb_world.h declare (checked against the built libraries by tests/test_abi.py)
def declared_symbols(include_dir):
    import re, os
    names = []
    for h in ("kjb.h", "kjb_world.h"):
        src = open(os.path.join(include_dir, h)).read()
        names += re.findall(r"\b(kjb_[a-z0-9_]+)\s*\(", src)
    return sorted(set(names))
