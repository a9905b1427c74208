"""Drive one pass at a time through the C-ABI on host arrays: the harness of the per-pass reference tests (`test_taa_reference.py`,
`test_rtr_reference.py`).

A `Runner` owns one context of one backend (kjb_create, kjb_image_alloc/upload, kjb_set_frame_constants, the pass, kjb_image_download)
and is driven by a pass table {name: (entry point, image bindings in kjb.h order, float4 constant count, host int32 pointer fields)}.
The struct it hands the pass is images, then float4s, then `const int32_t*` fields: the order every pass struct of kjb.h uses.
"""
import ctypes as C
import numpy as np

from kajiya_b200._abi import Image, FMT

F16, SNORM, DEPTH, RG16, R16 = FMT["RGBA16_FLOAT"], FMT["RGBA16_SNORM"], FMT["R32_FLOAT"], FMT["RG16_FLOAT"], FMT["R16_FLOAT"]
R11G11B10, A2R10G10B10, RGBA32F, R8 = FMT["R11G11B10_UFLOAT"], FMT["A2R10G10B10_UNORM"], FMT["RGBA32_FLOAT"], FMT["R8_UNORM"]
NP = {F16: (np.float16, 4), SNORM: (np.int16, 4), DEPTH: (np.float32, 1), RG16: (np.float16, 2), R16: (np.float16, 1),
      R11G11B10: (np.uint32, 1), A2R10G10B10: (np.uint32, 1), RGBA32F: (np.float32, 4), R8: (np.uint8, 1)}

VIEW_MATRICES = ["view_to_clip", "clip_to_view", "view_to_sample", "sample_to_view", "world_to_view", "view_to_world", "clip_to_prev_clip",
                 "prev_view_to_prev_clip", "prev_clip_to_prev_view", "prev_world_to_prev_view", "prev_view_to_prev_world"]


def _args(images, floats=0, pointers=()):
    fields = ([(n, Image) for n in images] + [(f"f{i}", C.c_float * 4) for i in range(floats)]
              + [(n, C.POINTER(C.c_int32)) for n in pointers])
    return type("Args", (C.Structure,), {"_fields_": fields})


def frame_constants(pre_exposure_delta=1.0, delta_time_seconds=1.0 / 60.0, sample_offset_pixels=(0.0, 0.0), frame_index=0, view=None):
    """kjb_frame_constants (1216 bytes, kjb.h): the view block from `view` ({name: 4x4 [row, col]}, see `view_constants`; zero without
    it), sample_offset_pixels, frame_index, delta_time_seconds and pre_exposure_delta; every other field zero."""
    fc = np.zeros(1216 // 4, np.float32)
    if view is not None:
        for i, n in enumerate(VIEW_MATRICES):
            fc[16 * i:16 * i + 16] = np.asarray(view[n], np.float32).T.ravel()   # glam column-major: element (r, c) at c * 4 + r
    fc[176:178] = sample_offset_pixels      # view_constants.sample_offset_pixels: after 11 mat4
    fc[184:185].view(np.uint32)[0] = frame_index   # after sun_direction[4]
    fc[185] = delta_time_seconds
    fc[198] = pre_exposure_delta            # after ..., sky_ambient[4], pre_exposure, pre_exposure_prev
    return fc


def view_constants(w, h, frame, pos, prev_pos, rot=(0.0, 0.0, 0.0, 1.0)):
    """The view block the frame driver builds for a `w` x `h` frame `frame` with the camera at `pos` (previously at `prev_pos`): the
    camera matrices and Halton jitter of `camera_reference.py`, which `test_host_mirror.py` checks against the driver (camera.rs:71-125,
    world_renderer.rs:425-428, 1001-1108).  Returns ({name: 4x4 [row, col]}, sample_offset_pixels)."""
    from camera_reference import camera, view_block
    v, off, _ = view_block(camera(pos, rot, w, h), camera(prev_pos, rot, w, h), frame, w, h)
    return v, (float(off[0]), float(off[1]))


def extent4(w, h):
    return [float(w), float(h), float(np.float32(1) / np.float32(w)), float(np.float32(1) / np.float32(h))]


class Runner:
    """One context of one backend; runs one pass on host arrays and returns its outputs as raw host arrays."""

    def __init__(self, lib, passes):
        self.lib, self.passes, d = lib, passes, lib.dll
        self.ctx = C.c_void_p()
        assert d.kjb_create(0 if lib.backend.startswith("cuda") else -1, C.byref(self.ctx)) == 0
        d.kjb_set_frame_constants.restype = C.c_int
        d.kjb_set_frame_constants.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]
        d.kjb_set_scissor.restype = C.c_int
        d.kjb_set_scissor.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
        for entry, *_ in passes.values():
            getattr(d, entry).restype = C.c_int
            getattr(d, entry).argtypes = [C.c_void_p, C.c_void_p]

    def err(self):
        return self.lib.dll.kjb_last_error(self.ctx).decode()

    def close(self):
        self.lib.dll.kjb_destroy(self.ctx)

    def run(self, pass_name, inputs, outputs, consts=(), fc=None, scissor=None, sentinel=None, pointers=None):
        """inputs: {binding: raw array (H, W, C) of the format's numpy type, format}; outputs: {binding: (w, h, format)};
        pointers: {field: int32 host array} for the pass's `const int32_t*` fields."""
        d, ctx = self.lib.dll, self.ctx
        entry, bindings, nf, *rest = self.passes[pass_name]
        ptr_fields = rest[0] if rest else ()
        fc = frame_constants() if fc is None else fc
        assert d.kjb_set_frame_constants(ctx, fc.ctypes.data, None, 0) == 0, self.err()
        imgs, keep = {}, []
        try:
            for b, (arr, fmt) in inputs.items():
                img = Image()
                assert d.kjb_image_alloc(ctx, arr.shape[1], arr.shape[0], 1, fmt, C.byref(img)) == 0, self.err()
                imgs[b] = img
                arr = np.ascontiguousarray(arr)
                keep.append(arr)
                assert d.kjb_image_upload(ctx, C.byref(img), arr.ctypes.data) == 0, self.err()
            for b, (w, h, fmt) in outputs.items():
                img = Image()
                assert d.kjb_image_alloc(ctx, w, h, 1, fmt, C.byref(img)) == 0, self.err()
                imgs[b] = img
                if sentinel is not None:
                    dt, c = NP[fmt]
                    fill = np.full(h * w * c * np.dtype(dt).itemsize, sentinel, np.uint8)
                    keep.append(fill)
                    assert d.kjb_image_upload(ctx, C.byref(img), fill.ctypes.data) == 0, self.err()
            args = _args(bindings, nf, ptr_fields)()
            for b in bindings:
                setattr(args, b, imgs.get(b, Image()))
            for i, c4 in enumerate(consts):
                getattr(args, f"f{i}")[:] = c4
            for p in ptr_fields:
                a = np.ascontiguousarray((pointers or {})[p], np.int32)
                keep.append(a)
                setattr(args, p, a.ctypes.data_as(C.POINTER(C.c_int32)))
            try:
                if scissor is not None:
                    assert d.kjb_set_scissor(ctx, *scissor) == 0, self.err()
                assert getattr(d, entry)(ctx, C.byref(args)) == 0, self.err()
            finally:
                if scissor is not None:
                    d.kjb_set_scissor(ctx, 0, 0)
            got = {}
            for b, (w, h, fmt) in outputs.items():
                dt, c = NP[fmt]
                out = np.empty((h, w, c), dt)
                assert d.kjb_image_download(ctx, C.byref(imgs[b]), out.ctypes.data) == 0, self.err()
                got[b] = out
            assert d.kjb_sync(ctx) == 0, self.err()
            return got
        finally:
            d.kjb_sync(ctx)   # the uploads read `keep` and the downloads write `got` until the stream drains
            for img in imgs.values():
                d.kjb_image_free(ctx, C.byref(img))


class Runners:
    """One Runner per backend, created on first use and destroyed with the module's tests."""

    def __init__(self, passes):
        self.passes, self._by_path = passes, {}

    def __call__(self, lib):
        if lib.path not in self._by_path:
            self._by_path[lib.path] = Runner(lib, self.passes)
        return self._by_path[lib.path]

    def close(self):
        for r in self._by_path.values():
            r.close()
        self._by_path.clear()
