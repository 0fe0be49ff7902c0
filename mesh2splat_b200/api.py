"""Host-side mirror of the reference's interface for the conversion path, over the C ABI.

Reference surface (src/utils/SceneManager.hpp:18-20, src/renderer/renderPasses/RenderPass.hpp:10-28,
src/renderer/RenderContext.hpp:28-124):

    SceneManager::loadModel(path, parentFolder)      -> SceneManager.loadModel / .setScene
    ConversionPass::execute(RenderContext&)          -> ConversionPass.execute(renderContext)
    SceneManager::exportPly(outPath, exportFormat)   -> SceneManager.exportPly
    SceneManager::loadPly(filePath)                  -> SceneManager.loadPly (parsers::loadPlyFile on the GPU)

plus the plain functional form `Context.convert(...)`.  torch is used only to own device buffers
(torch.empty(..., device="cuda")) and pinned host buffers; every computation is a call into
libm2s.so.
"""
from __future__ import annotations

import ctypes as C
from contextlib import contextmanager
from dataclasses import dataclass

import numpy as np

from . import _abi
from ._lib import M2SError, check, lib


def _torch():
    import torch  # noqa: WPS433 (lazy: the ABI layer itself does not need torch)
    return torch


def _binned_pass(dev, max_pairs, n, draw, draw_enqueue):
    """The two forms of a binned pass (splat draw, mesh depth, shadow map); returns (drawn, pairs).  max_pairs None:
    draw(pairs) synchronously, all n items drawn.  Otherwise draw_enqueue(max_pairs, d_pairs, d_drawn, stream) on torch's
    current stream with that pair budget, then the pair total and the drawn prefix read back."""
    torch = _torch()
    if max_pairs is None:
        torch.cuda.synchronize(dev)   # the buffers torch filled are ready before the context stream reads them
        pairs = C.c_uint64(0)
        check(draw(C.byref(pairs)))
        return n, int(pairs.value)
    out = torch.zeros(4, dtype=torch.int32, device=dev)   # pairs (uint64) | drawn (uint32)
    check(draw_enqueue(max_pairs, out.data_ptr(), out[2:].data_ptr(), torch.cuda.current_stream(dev).cuda_stream))
    torch.cuda.synchronize(dev)
    o = out.cpu().numpy()
    return int(o[2]), int(o[:2].view(np.uint64)[0])


def _gbuffer(dev, width: int, height: int, targets, gbuffer):
    """The m2s_gbuffer of the named targets, each the caller's tensor in `gbuffer` or a new one; (struct, {name: tensor})."""
    torch = _torch()
    gbuffer = dict(gbuffer or {})
    g = _abi.m2s_gbuffer()
    for name, dt in _abi.GBUFFER_TARGETS:
        if name not in targets:
            continue
        if name not in gbuffer:
            gbuffer[name] = torch.empty(width * height * 4, dtype=torch.int16 if dt == np.float16 else torch.uint8, device=dev)
        setattr(g, name, gbuffer[name].data_ptr())
    return g, gbuffer


def _gbuffer_of(tensors: dict):
    """The m2s_gbuffer of {target name: device tensor or None}."""
    g = _abi.m2s_gbuffer()
    for name, t in tensors.items():
        if t is not None:
            setattr(g, name, t.data_ptr())
    return g


def _gbuffer_images(gbuffer: dict, width: int, height: int, targets) -> dict:
    """The drawn targets as {name: numpy array (height, width, 4)}, float16 or uint8."""
    torch = _torch()
    images = {}
    for name, dt in _abi.GBUFFER_TARGETS:
        if name in targets:
            raw = gbuffer[name].view(torch.uint8)[: width * height * 4 * np.dtype(dt).itemsize]
            images[name] = raw.cpu().numpy().view(dt).reshape(height, width, 4).copy()
    return images


class DeviceScene:
    """Device-resident scene (triangles, primitive table, mip chains): what loadModel leaves on the
    GPU in the reference (VBOs + GL textures)."""

    def __init__(self, ctx: "Context", handle: int, scene: _abi.Scene):
        self.ctx, self.handle = ctx, handle
        self.primitive_count = len(scene.primitives)
        self.triangle_count = scene.triangle_count
        self.texture_shapes = [t.shape[:2] for t in scene.textures]

    def read_mip(self, texture: int, level: int) -> np.ndarray:
        h, w = self.texture_shapes[texture]
        buf = np.zeros((h, w, 4), np.uint8)
        ow, oh = C.c_uint32(0), C.c_uint32(0)
        check(lib().m2s_scene_read_mip(self.ctx.handle, self.handle, texture, level, buf.ctypes.data,
                                       C.byref(ow), C.byref(oh)))
        return buf.reshape(-1)[: ow.value * oh.value * 4].reshape(oh.value, ow.value, 4).copy()

    def h2d_bytes(self) -> int:
        return int(lib().m2s_scene_h2d_bytes(self.handle))

    def r_small_max(self) -> float:
        """The largest density at which every triangle's candidate box is certainly small (m2s_debug_scene_r_small_max):
        PACKED56 conversions up to it end in the raster kernel.  0 for scenes uploaded in part (no slim triangle stream)."""
        fn = lib().m2s_debug_scene_r_small_max
        fn.restype = C.c_float
        fn.argtypes = [C.c_void_p]
        return float(fn(self.handle))

    def free(self):
        if self.handle:
            lib().m2s_scene_free(self.ctx.handle, self.handle)
            self.handle = 0

    def __del__(self):
        try:
            self.free()
        except Exception:  # noqa: BLE001
            pass


@dataclass
class ConvertOutput:
    data: object            # torch.uint8 tensor on the device, capacity * stride bytes
    keys: object            # torch.int64 tensor (fragment identity) or None
    total: int              # fragments generated (reference: numberOfGaussians)
    written: int            # records stored = min(total, cap)
    cap: int
    device_ms: float
    layout: int
    overflow: bool

    def numpy(self) -> np.ndarray:
        stride = _abi.STRIDES[self.layout]
        raw = self.data[: self.written * stride].cpu().numpy()
        return raw.view(_abi.record_dtype(self.layout))

    def keys_numpy(self):
        return None if self.keys is None else self.keys[: self.written].cpu().numpy().view(np.uint64)


class Context:
    """One per GPU (m2s_ctx)."""

    def __init__(self, device: int = 0):
        h = C.c_void_p(0)
        check(lib().m2s_ctx_create(device, C.byref(h)))
        self.handle = h.value
        self.device = device
        self.sm_count = lib().m2s_ctx_sm_count(self.handle)

    def close(self):
        if getattr(self, "handle", 0):
            lib().m2s_ctx_destroy(self.handle)
            self.handle = 0

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    # ---- inputs ----
    def upload(self, scene: _abi.Scene) -> DeviceScene:
        cs, keep = scene.c_struct()
        h = C.c_void_p(0)
        check(lib().m2s_scene_upload(self.handle, C.byref(cs), C.byref(h)))
        del keep
        return DeviceScene(self, h.value, scene)

    def upload_range(self, scene: _abi.Scene, layout: int, first_triangle: int, triangle_count: int, c_scene=None) -> DeviceScene:
        """One shard (m2s_scene_upload_range): the triangle range at its global indices + only the texture rows it samples."""
        cs, keep = c_scene if c_scene is not None else scene.c_struct()
        h = C.c_void_p(0)
        check(lib().m2s_scene_upload_range(self.handle, C.byref(cs), layout, first_triangle, triangle_count, C.byref(h)))
        del keep
        return DeviceScene(self, h.value, scene)

    # ---- the hot path ----
    @staticmethod
    def default_capacity(primitive_count: int, resolution: int, max_gaussians: int, flags: int) -> int:
        if max_gaussians:
            return max_gaussians
        if flags & _abi.FLAG_UNCAPPED:
            return 6 * resolution * resolution * max(1, primitive_count)
        return _abi.reference_capacity(resolution, primitive_count)

    def convert(self, dscene: DeviceScene, resolution: int, layout: int = _abi.LAYOUT_REF96,
                gaussian_std: float = 0.65, max_gaussians: int = 0, flags: int = 0, first_triangle: int = 0,
                triangle_count: int = 0, capacity: int | None = None, want_keys: bool = False,
                out=None, keys=None, allow_overflow: bool = True, row_begin: int = 0, row_end: int = 0) -> ConvertOutput:
        torch = _torch()
        stride = _abi.STRIDES[layout]
        if capacity is None:
            capacity = self.default_capacity(dscene.primitive_count, resolution, max_gaussians, flags)
        dev = torch.device("cuda", self.device)
        if out is None:
            out = torch.empty(max(1, capacity) * stride, dtype=torch.uint8, device=dev)
        if want_keys and keys is None:
            keys = torch.empty(max(1, capacity), dtype=torch.int64, device=dev)
        p = _abi.make_params(resolution, layout, gaussian_std, max_gaussians, flags, first_triangle, triangle_count,
                             row_begin, row_end)
        res = _abi.m2s_result()
        st = check(lib().m2s_convert(self.handle, dscene.handle, C.byref(p), out.data_ptr(), capacity,
                                     keys.data_ptr() if keys is not None else None, C.byref(res)),
                   allow=(_abi.M2S_E_CAPACITY,) if allow_overflow else ())
        return ConvertOutput(out, keys, int(res.total), int(res.written), int(res.cap), float(res.device_ms), layout,
                             st == _abi.M2S_E_CAPACITY)

    @staticmethod
    @contextmanager
    def single_launch_off():
        """Within the block, conversions that could end in the raster kernel launch the fragment kernel as well
        (m2s_debug_set_single_off): the two-kernel route that the single launch is compared against."""
        fn = lib().m2s_debug_set_single_off
        fn.argtypes = [C.c_int]
        fn(1)
        try:
            yield
        finally:
            fn(0)

    def convert_plan(self, dscene: DeviceScene, resolution: int, layout: int = _abi.LAYOUT_REF96, capacity: int = 0,
                     max_gaussians: int = 0, flags: int = 0, first_triangle: int = 0,
                     triangle_count: int = 0) -> _abi.m2s_convert_plan:
        """The launch plan convert() makes for the same arguments (m2s_debug_convert_plan): grid, work units, item
        sizes, effective cap and the raster kernel's route (multi_round, direct_ok, claim_late)."""
        L = lib()
        fn = L.m2s_debug_convert_plan
        fn.restype = C.c_int
        fn.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(_abi.m2s_params), C.c_uint64, C.POINTER(_abi.m2s_convert_plan)]
        p = _abi.make_params(resolution, layout, 0.65, max_gaussians, flags, first_triangle, triangle_count)
        plan = _abi.m2s_convert_plan()
        check(fn(self.handle, dscene.handle, C.byref(p), capacity, C.byref(plan)))
        return plan

    def codec_eval(self, fn: int, x, arg: float = 1.0, out=None):
        """One function of m2s_codec.cuh (_abi.CODEC_*) applied elementwise to a float32 device tensor on torch's current
        stream (m2s_debug_codec_eval): the encodings the conversion and the .ply writer use, the decodings the loader
        uses.  arg: the scale multiplier of CODEC_LOG_SCALE."""
        torch = _torch()
        fn_c = lib().m2s_debug_codec_eval
        fn_c.restype = C.c_int
        fn_c.argtypes = [C.c_void_p, C.c_uint32, C.c_float, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
        x = x.contiguous()
        if out is None:
            out = torch.empty_like(x)
        check(fn_c(self.handle, fn, arg, x.data_ptr(), x.numel(), out.data_ptr(), torch.cuda.current_stream(x.device).cuda_stream))
        return out

    def convert_enqueue(self, dscene: DeviceScene, params: _abi.m2s_params, out, capacity: int, keys=None,
                        total=None, stream: int = 0) -> None:
        """Enqueue only (no synchronisation); out/keys/total are torch device tensors."""
        check(lib().m2s_convert_enqueue(self.handle, dscene.handle, C.byref(params), out.data_ptr(), capacity,
                                        keys.data_ptr() if keys is not None else None,
                                        total.data_ptr() if total is not None else None, stream or None))

    def prepass(self, records, count: int, layout: int, world_to_view, view_to_clip, model_to_world, resolution, near_far,
                std_dev: float, render_mode: int = 0, quads=None, depths=None, mesh_depth=None, sh=None, sh_degree=None):
        """GaussiansPrepass::execute on device-resident records (a torch uint8 tensor, e.g. ConvertOutput.data): returns
        (quads [m, 24] float32, depths [m] float32) as numpy arrays, in atomic arrival order (m2s_prepass).
        quads / depths: optional caller-owned device tensors of at least count * 96 bytes / count floats.
        mesh_depth: None, or a float32 device tensor (H, W) from mesh_depth(..., depth=...): the prepass with the mesh
        depth test (m2s_prepass_mesh_depth).
        sh / sh_degree: view-dependent colour from a loaded .ply's SH rest coefficients (m2s_prepass_sh; layouts VIEW_PLY
        and VIEW_PLY_PBR).  sh: the (count, 12 | 24 | 48) float32 device tensor of ply_read_sh, whose width sets the
        buffer's degree; sh_degree: the degree evaluated (default the buffer's).  Both None: m2s_prepass."""
        import torch
        dev = records.device
        if quads is None:
            quads = torch.empty(max(1, count) * _abi.QUAD_BYTES, dtype=torch.uint8, device=dev)
        if depths is None:
            depths = torch.empty(max(1, count), dtype=torch.float32, device=dev)
        p = _abi.make_prepass_params(world_to_view, view_to_clip, model_to_world, resolution, near_far, std_dev, render_mode, layout)
        valid = C.c_uint32(0)
        if sh is not None or sh_degree is not None:
            if mesh_depth is not None:
                raise ValueError("sh and mesh_depth do not combine (a loaded .ply never reads the mesh depth map)")
            buffer_degree = 0
            if sh is not None:
                degrees = {f: d for d, f in _abi.SH_FLOATS.items() if f}
                if sh.dim() != 2 or sh.shape[1] not in degrees or sh.dtype != torch.float32 or sh.device != dev or not sh.is_contiguous():
                    raise ValueError("sh must be a contiguous (count, 12 | 24 | 48) float32 tensor on the records' device")
                buffer_degree = degrees[sh.shape[1]]
            torch.cuda.synchronize(dev)   # the coefficients torch holds are ready before the context stream reads them
            check(lib().m2s_prepass_sh(self.handle, records.data_ptr(), count, C.byref(p), sh.data_ptr() if sh is not None else None,
                                       buffer_degree, buffer_degree if sh_degree is None else int(sh_degree), quads.data_ptr(),
                                       depths.data_ptr(), C.byref(valid)))
        elif mesh_depth is None:
            check(lib().m2s_prepass(self.handle, records.data_ptr(), count, C.byref(p), quads.data_ptr(), depths.data_ptr(), C.byref(valid)))
        else:
            if (mesh_depth.dim() != 2 or mesh_depth.dtype != torch.float32 or mesh_depth.device != dev
                    or not mesh_depth.is_contiguous()):
                raise ValueError("mesh_depth must be a contiguous (height, width) float32 tensor on the records' device")
            h, w = mesh_depth.shape
            torch.cuda.synchronize(dev)   # the map torch holds is ready before the context stream reads it
            check(lib().m2s_prepass_mesh_depth(self.handle, records.data_ptr(), count, C.byref(p), mesh_depth.data_ptr(), w, h,
                                               quads.data_ptr(), depths.data_ptr(), C.byref(valid)))
        m = int(valid.value)
        return quads[: m * _abi.QUAD_BYTES].cpu().numpy().view(np.float32).reshape(m, 24).copy(), depths[:m].cpu().numpy().copy()

    def depth_sort(self, quads, depths, count: int, d_count=None, sorted_quads=None, order=None, draw=None):
        """RadixSortPass::execute on the prepass output (m2s_depth_sort): the quads (a torch uint8 device tensor of
        count * 96 bytes) stably sorted by the uint32 bits of their view depths (a float32 device tensor of count values).
        Returns (sorted_quads [n, 24] float32, order [n] uint32, draw [5] uint32) as numpy arrays, n = count or
        min(count, d_count[0]).  d_count: optional uint32/int32 device tensor (the prepass's valid counter); with it the
        call is enqueued on torch's current stream (m2s_depth_sort_enqueue).  sorted_quads / order / draw: optional
        caller-owned device tensors of at least count * 96 bytes / count and 5 32-bit words."""
        torch = _torch()
        dev = quads.device
        if sorted_quads is None:
            sorted_quads = torch.empty(max(1, count) * _abi.QUAD_BYTES, dtype=torch.uint8, device=dev)
        if order is None:
            order = torch.empty(max(1, count), dtype=torch.int32, device=dev)
        if draw is None:
            draw = torch.empty(5, dtype=torch.int32, device=dev)
        if d_count is None:
            torch.cuda.synchronize(dev)   # the buffers torch filled are ready before the context stream reads them
            check(lib().m2s_depth_sort(self.handle, quads.data_ptr(), depths.data_ptr(), count, sorted_quads.data_ptr(),
                                       order.data_ptr(), draw.data_ptr()))
        else:
            check(lib().m2s_depth_sort_enqueue(self.handle, quads.data_ptr(), depths.data_ptr(), count, d_count.data_ptr(),
                                               sorted_quads.data_ptr(), order.data_ptr(), draw.data_ptr(),
                                               torch.cuda.current_stream(dev).cuda_stream))
            torch.cuda.synchronize(dev)
        d = draw[:5].cpu().numpy().view(np.uint32).copy()
        n = int(d[1])
        return (sorted_quads[: n * _abi.QUAD_BYTES].cpu().numpy().view(np.float32).reshape(n, 24).copy(),
                order[:n].cpu().numpy().view(np.uint32).copy(), d)

    def splat_draw(self, sorted_quads, count: int, width: int, height: int, render_mode: int = 0, d_draw=None,
                   targets=tuple(name for name, _ in _abi.GBUFFER_TARGETS), max_pairs: int | None = None, gbuffer=None):
        """GaussianSplattingPass::execute on the sorted quads (a torch uint8 device tensor of count * 96 bytes): the
        G-buffer as {target name: numpy array (height, width, 4)}, float16 for position / normal / depth and uint8 for
        albedo / metallic_roughness, row 0 = the bottom row; plus (drawn, pairs).  targets: the names to draw.
        max_pairs None: m2s_splat_draw (all quads drawn).  Otherwise m2s_splat_draw_enqueue on torch's current stream with
        that pair budget, d_draw (optional int32 device tensor, the sort's draw command) limiting n.  gbuffer: optional
        {name: caller-owned device tensor of width * height * 4 elements} for the drawn targets."""
        dev = sorted_quads.device
        g, gbuffer = _gbuffer(dev, width, height, targets, gbuffer)
        p = _abi.m2s_splat_params(width, height, render_mode)
        drawn, npairs = _binned_pass(
            dev, max_pairs, count,
            lambda pairs: lib().m2s_splat_draw(self.handle, sorted_quads.data_ptr(), count, C.byref(p), C.byref(g), pairs),
            lambda *budget: lib().m2s_splat_draw_enqueue(self.handle, sorted_quads.data_ptr(), count,
                                                         d_draw.data_ptr() if d_draw is not None else None, C.byref(p),
                                                         C.byref(g), *budget))
        return _gbuffer_images(gbuffer, width, height, targets), drawn, npairs

    def mesh_depth(self, dscene: DeviceScene, world_to_view, view_to_clip, model_to_world, width: int, height: int,
                   max_pairs: int | None = None, depth=None):
        """DepthPrepass::execute on an uploaded scene: returns (map (height, width) float32 numpy, row 0 = window y 0,
        drawn, pairs).  max_pairs None: m2s_mesh_depth (every triangle drawn).  Otherwise m2s_mesh_depth_enqueue on torch's
        current stream with that pair budget.  depth: optional caller-owned float32 device tensor of at least
        width * height values (pass it on to prepass(mesh_depth=...) viewed as (height, width))."""
        torch = _torch()
        dev = torch.device("cuda", self.device)
        if depth is None:
            depth = torch.empty(width * height, dtype=torch.float32, device=dev)
        elif depth.dtype != torch.float32 or depth.device != dev or not depth.is_contiguous() or depth.numel() < width * height:
            raise ValueError("depth must be a contiguous float32 tensor of at least width * height values on the context's device")
        p = _abi.make_mesh_depth_params(world_to_view, view_to_clip, model_to_world, width, height)
        drawn, npairs = _binned_pass(
            dev, max_pairs, dscene.triangle_count,
            lambda pairs: lib().m2s_mesh_depth(self.handle, dscene.handle, C.byref(p), depth.data_ptr(), pairs),
            lambda *budget: lib().m2s_mesh_depth_enqueue(self.handle, dscene.handle, C.byref(p), depth.data_ptr(), *budget))
        return depth.reshape(-1)[: width * height].cpu().numpy().reshape(height, width).copy(), drawn, npairs

    def mesh_render(self, dscene: DeviceScene, world_to_view, view_to_clip, model_to_world, width: int, height: int, near_far,
                    render_mode: int = 0, targets=tuple(name for name, _ in _abi.GBUFFER_TARGETS), max_pairs: int | None = None,
                    gbuffer=None):
        """MeshRenderPass::execute on an uploaded scene: the mesh G-buffer as {target name: numpy array (height, width, 4)}
        (float16 for position / normal / depth, uint8 for albedo / metallic_roughness, row 0 = the bottom row), plus
        (drawn, pairs).  targets: the names to draw.  max_pairs None: m2s_mesh_render (every triangle drawn).  Otherwise
        m2s_mesh_render_enqueue on torch's current stream with that pair budget.  gbuffer: optional {name: caller-owned
        device tensor of width * height * 4 elements} for the drawn targets (pass them on to deferred_light_split)."""
        torch = _torch()
        dev = torch.device("cuda", self.device)
        g, gbuffer = _gbuffer(dev, width, height, targets, gbuffer)
        p = _abi.make_mesh_render_params(world_to_view, view_to_clip, model_to_world, width, height, near_far, render_mode)
        drawn, npairs = _binned_pass(
            dev, max_pairs, dscene.triangle_count,
            lambda pairs: lib().m2s_mesh_render(self.handle, dscene.handle, C.byref(p), C.byref(g), pairs),
            lambda *budget: lib().m2s_mesh_render_enqueue(self.handle, dscene.handle, C.byref(p), C.byref(g), *budget))
        return _gbuffer_images(gbuffer, width, height, targets), drawn, npairs

    def shadow_map(self, records, count: int, layout: int, model_to_world, light_position, near_far, resolution, std_dev: float,
                   size: int = 1024, max_pairs: int | None = None, d_count=None, cube=None, light_quads=None):
        """GaussianShadowPass::execute on device-resident records (a torch uint8 tensor, e.g. ConvertOutput.data): returns
        (cube [6, S, S] float32, light records [count, 8] float32 (word 7: face bits), drawn, pairs) as numpy values.
        max_pairs None: m2s_shadow_map (all records drawn).  Otherwise m2s_shadow_map_enqueue on torch's current stream
        with that pair budget and d_count (optional uint64 device tensor, the conversion's counter) limiting n.  cube /
        light_quads: optional caller-owned device tensors of at least 6 S^2 floats / count * 32 bytes."""
        torch = _torch()
        dev = records.device
        if cube is None:
            cube = torch.empty(6 * size * size, dtype=torch.float32, device=dev)
        if light_quads is None:
            light_quads = torch.empty(max(1, count) * _abi.LIGHT_RECORD_BYTES, dtype=torch.uint8, device=dev)
        p = _abi.make_shadow_params(model_to_world, light_position, near_far, resolution, std_dev, layout, size)
        drawn, npairs = _binned_pass(
            dev, max_pairs, count,
            lambda pairs: lib().m2s_shadow_map(self.handle, records.data_ptr(), count, C.byref(p), cube.data_ptr(),
                                               light_quads.data_ptr(), pairs),
            lambda *budget: lib().m2s_shadow_map_enqueue(self.handle, records.data_ptr(), count,
                                                         d_count.data_ptr() if d_count is not None else None, C.byref(p),
                                                         cube.data_ptr(), light_quads.data_ptr(), *budget))
        lq = light_quads.view(torch.uint8)[: count * _abi.LIGHT_RECORD_BYTES].cpu().numpy().view(np.float32).reshape(count, 8).copy()
        return cube[: 6 * size * size].cpu().numpy().reshape(6, size, size).copy(), lq, drawn, npairs

    def deferred_light(self, gbuffer: dict, cube, width: int, height: int, render_mode: int = 6, light_position=(0.0, 0.0, 0.0),
                       light_color=(1.0, 1.0, 1.0), light_intensity: float = 1.0, cam_pos=(0.0, 0.0, 0.0), far_plane: float = 100.0,
                       shadow_size: int = 1024, image=None, enqueue: bool = False):
        """GaussianRelightingPass::execute: the RGBA8 image (height, width, 4) uint8, row 0 = the bottom row, as numpy.
        gbuffer: {target name: device tensor} (the splat draw's targets; the mode's required ones must be present);
        cube: device float32 tensor of 6 S^2 values or None (modes 0-5).  enqueue: m2s_deferred_light_enqueue on torch's
        current stream instead of the synchronous m2s_deferred_light.  image: optional caller-owned device tensor of
        width * height * 4 bytes."""
        return self._light((gbuffer,), cube, width, height, image, enqueue, lib().m2s_deferred_light_enqueue, lib().m2s_deferred_light,
                           _abi.make_light_params(width, height, render_mode, light_position, light_color, light_intensity, cam_pos,
                                                  far_plane, shadow_size))

    def deferred_light_split(self, splat_gbuffer: dict, mesh_gbuffer: dict, cube, width: int, height: int, split_position: float,
                             render_mode: int = 6, light_position=(0.0, 0.0, 0.0), light_color=(1.0, 1.0, 1.0),
                             light_intensity: float = 1.0, cam_pos=(0.0, 0.0, 0.0), far_plane: float = 100.0, shadow_size: int = 1024,
                             image=None, enqueue: bool = False):
        """GaussianRelightingPass::execute in split screen: the mesh G-buffer lit left of int(split_position * width),
        the splat G-buffer right of it, the two divider columns white; the RGBA8 image (height, width, 4) as numpy.
        Everything else as deferred_light."""
        return self._light((splat_gbuffer, mesh_gbuffer), cube, width, height, image, enqueue, lib().m2s_deferred_light_split_enqueue,
                           lib().m2s_deferred_light_split,
                           _abi.make_light_params(width, height, render_mode, light_position, light_color, light_intensity, cam_pos,
                                                  far_plane, shadow_size), float(split_position))

    def _light(self, gbuffers, cube, width, height, image, enqueue, light_enqueue, light, params, *extra):
        """Both lighting calls: light(ctx, *gbuffers, cube, params, *extra, image), or light_enqueue with torch's current
        stream appended; the image read back as numpy."""
        torch = _torch()
        dev = next((t.device for gb in gbuffers for t in gb.values() if t is not None), cube.device if cube is not None else None)
        if image is None:
            image = torch.empty(width * height * 4, dtype=torch.uint8, device=dev)
        args = (self.handle, *(C.byref(_gbuffer_of(gb)) for gb in gbuffers), cube.data_ptr() if cube is not None else None, C.byref(params),
                *extra, image.data_ptr())
        if enqueue:
            check(light_enqueue(*args, torch.cuda.current_stream(dev).cuda_stream))
        else:
            torch.cuda.synchronize(dev)
            check(light(*args))
        torch.cuda.synchronize(dev)
        return image.view(torch.uint8)[: width * height * 4].cpu().numpy().reshape(height, width, 4).copy()

    def compare_images(self, a, b, width: int, height: int, cover_a=None, cover_b=None, cover_min: int = 128, ssim_map=None,
                       enqueue: bool = False) -> dict:
        """How closely image b reproduces image a (m2s_image_compare): SSIM over the valid 11 x 11 windows, squared error
        and coverage of two RGBA8 device tensors of width * height * 4 bytes (e.g. the lit mesh and the lit splats of one
        frame).  cover_a / cover_b: optional RGBA8 device tensors whose alpha >= cover_min marks a pixel covered (e.g. the
        albedo targets of the two G-buffers).  ssim_map: optional float32 device tensor of at least (width - 10) *
        (height - 10) values, filled with the per-window SSIM (row 0 = window y 5).  enqueue: m2s_image_compare_enqueue on
        torch's current stream instead of the synchronous call.  Returns the totals (windows, covered_windows,
        pixels_both, pixels_a_only, pixels_b_only, sq_err, sq_err_covered, ssim_sum, ssim_covered_sum) and the derived
        psnr, ssim, psnr_covered and ssim_covered."""
        torch = _torch()
        dev = a.device
        p = _abi.m2s_compare_params(width, height, cover_min)
        ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
        args = (self.handle, ptr(a), ptr(b), ptr(cover_a), ptr(cover_b), C.byref(p))
        if enqueue:
            d_result = torch.zeros(C.sizeof(_abi.m2s_compare_result), dtype=torch.uint8, device=dev)
            check(lib().m2s_image_compare_enqueue(*args, d_result.data_ptr(), ptr(ssim_map), torch.cuda.current_stream(dev).cuda_stream))
            torch.cuda.synchronize(dev)
            r = _abi.m2s_compare_result.from_buffer_copy(d_result.cpu().numpy().tobytes())
        else:
            r = _abi.m2s_compare_result()
            torch.cuda.synchronize(dev)   # the images torch filled are ready before the context stream reads them
            check(lib().m2s_image_compare(*args, C.byref(r), ptr(ssim_map)))
        return _abi.compare_result_dict(r, width * height)

    def render_3dgs(self, records, count: int, layout: int, world_to_view, view_to_clip, model_to_world, width: int, height: int,
                    near: float = 0.2, std_dev: float = 1.0, scale_modifier: float = 1.0, background=(0.0, 0.0, 0.0), sh=None,
                    sh_degree: int | None = None, targets=("rgba8", "rgba32f"), max_pairs: int | None = None, d_count=None,
                    images=None):
        """The standard 3DGS render (m2s_3dgs_render, graphdeco's forward pass) of device-resident records (a torch uint8
        tensor, e.g. ConvertOutput.data or ply_read's): returns ({target: device tensor}, drawn, pairs).  "rgba8" is a uint8
        tensor of width * height * 4 bytes (it feeds compare_images directly), "rgba32f" a float32 tensor of width * height
        * 4 values; row 0 = the bottom row.  targets: the names to draw.  sh / sh_degree: a loaded .ply's SH rest
        coefficients, as prepass (layouts VIEW_PLY and VIEW_PLY_PBR).  max_pairs None: m2s_3dgs_render (every survivor
        drawn).  Otherwise m2s_3dgs_render_enqueue on torch's current stream with that pair budget and d_count (optional
        uint64 device tensor) limiting n.  images: optional {target: caller-owned device tensor}."""
        torch = _torch()
        dev = records.device
        images = dict(images or {})
        for name, dt in (("rgba8", torch.uint8), ("rgba32f", torch.float32)):
            if name in targets and name not in images:
                images[name] = torch.empty(width * height * 4, dtype=dt, device=dev)
        images = {k: v for k, v in images.items() if k in targets}
        buffer_degree, sh_ptr = self._sh_buffer(sh, dev)
        degree = buffer_degree if sh_degree is None else int(sh_degree)
        p = _abi.make_3dgs_params(world_to_view, view_to_clip, model_to_world, width, height, near, std_dev, scale_modifier, background, layout)
        ptr = lambda name: images[name].data_ptr() if name in images else None  # noqa: E731
        drawn, npairs = _binned_pass(
            dev, max_pairs, count,
            lambda pairs: lib().m2s_3dgs_render(self.handle, records.data_ptr(), count, C.byref(p), sh_ptr, buffer_degree, degree,
                                                ptr("rgba32f"), ptr("rgba8"), pairs),
            lambda *budget: lib().m2s_3dgs_render_enqueue(self.handle, records.data_ptr(), count,
                                                          d_count.data_ptr() if d_count is not None else None, C.byref(p), sh_ptr,
                                                          buffer_degree, degree, ptr("rgba32f"), ptr("rgba8"), *budget))
        return images, drawn, npairs

    def gs3d_state(self) -> "Gs3dState":
        """A state of the 3DGS render's backward pass (m2s_3dgs_state): holds one forward pass of render_3dgs_grad until
        its backward.  Free it (or use it as a context manager) before the context."""
        return Gs3dState(self)

    def render_3dgs_grad(self, params, state: "Gs3dState", world_to_view, view_to_clip, model_to_world, width: int, height: int,
                         near: float = 0.2, scale_modifier: float = 1.0, background=(0.0, 0.0, 0.0), max_pairs: int | None = None):
        """The standard 3DGS render of PACKED56 gaussians as a differentiable torch operation: params is a (count, 14)
        float32 CUDA tensor (xyz, quaternion wxyz, log-scale, SH0, opacity logit; e.g. out.data[:n * 56].view(torch.float32)
        .view(n, 14)).  Returns the (height, width, 4) RGBA32F image (row 0 = the bottom row), bit for bit render_3dgs's.
        Its backward (m2s_3dgs_backward_enqueue on torch's current stream, no synchronisation) fills params.grad.
        max_pairs None: m2s_3dgs_render_grad (every survivor drawn; one read-back of the pair count); otherwise
        m2s_3dgs_render_grad_enqueue on torch's current stream with that pair budget.  The state keeps this forward pass
        until the next one that uses it; the backward of an older one raises."""
        p = _abi.make_3dgs_params(world_to_view, view_to_clip, model_to_world, width, height, near, 1.0, scale_modifier, background,
                                  _abi.LAYOUT_PACKED56)
        return _Render3dgsGrad.apply(params, self, state, p, max_pairs)

    def gs3d_preprocess(self, records, count: int, layout: int, world_to_view, view_to_clip, model_to_world, width: int, height: int,
                        near: float = 0.2, std_dev: float = 1.0, scale_modifier: float = 1.0, sh=None, sh_degree: int | None = None):
        """The 3DGS render's preprocess kernel alone (m2s_debug_3dgs_preprocess, not in m2s.h): (splat records [count, 12]
        float32, depth keys [count] uint32 (GS3D_CULLED for a culled record), survivors) as numpy values."""
        torch = _torch()
        dev = records.device
        fn = lib().m2s_debug_3dgs_preprocess
        fn.restype = C.c_int
        fn.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(_abi.m2s_3dgs_params), C.c_void_p, C.c_uint32, C.c_uint32,
                       C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32)]
        splats = torch.empty(max(1, count) * _abi.GS3D_SPLAT_FLOATS, dtype=torch.float32, device=dev)
        keys = torch.empty(max(1, count), dtype=torch.int32, device=dev)
        buffer_degree, sh_ptr = self._sh_buffer(sh, dev)
        p = _abi.make_3dgs_params(world_to_view, view_to_clip, model_to_world, width, height, near, std_dev, scale_modifier, (0, 0, 0), layout)
        survivors = C.c_uint32(0)
        torch.cuda.synchronize(dev)
        check(fn(self.handle, records.data_ptr(), count, C.byref(p), sh_ptr, buffer_degree, buffer_degree if sh_degree is None else int(sh_degree),
                 splats.data_ptr(), keys.data_ptr(), C.byref(survivors)))
        return (splats[: count * _abi.GS3D_SPLAT_FLOATS].cpu().numpy().reshape(count, _abi.GS3D_SPLAT_FLOATS).copy(),
                keys[:count].cpu().numpy().view(np.uint32).copy(), int(survivors.value))

    @staticmethod
    def _sh_buffer(sh, dev):
        """(buffer degree, device pointer) of an SH tensor as ply_read_sh returns it, (0, None) for None."""
        if sh is None:
            return 0, None
        torch = _torch()
        degrees = {f: d for d, f in _abi.SH_FLOATS.items() if f}
        if sh.dim() != 2 or sh.shape[1] not in degrees or sh.dtype != torch.float32 or sh.device != dev or not sh.is_contiguous():
            raise ValueError("sh must be a contiguous (count, 12 | 24 | 48) float32 tensor on the records' device")
        return degrees[sh.shape[1]], sh.data_ptr()

    def convert_timed(self, dscene: DeviceScene, params: _abi.m2s_params, out, capacity: int):
        """One conversion with an event between the two kernels (they do not overlap): (raster_ms, fragment_ms)."""
        a, b = C.c_float(0), C.c_float(0)
        check(lib().m2s_convert_timed(self.handle, dscene.handle, C.byref(params), out.data_ptr(), capacity, C.byref(a), C.byref(b)))
        return float(a.value), float(b.value)

    def convert_host(self, scene: _abi.Scene, resolution: int, layout: int = _abi.LAYOUT_REF96,
                     gaussian_std: float = 0.65, max_gaussians: int = 0, flags: int = 0, capacity: int | None = None,
                     want_keys: bool = False, out: np.ndarray | None = None, c_scene=None, keys: np.ndarray | None = None):
        """Host buffers in, host buffers out (m2s_convert_host). Returns (records, keys, result).
        out / keys: optional caller-owned host arrays (uint8, >= capacity * stride bytes / uint64, >= capacity)."""
        stride = _abi.STRIDES[layout]
        if capacity is None:
            capacity = self.default_capacity(len(scene.primitives), resolution, max_gaussians, flags)
        if out is None:
            out = np.empty(max(1, capacity) * stride, np.uint8)
        if want_keys and keys is None:
            keys = np.empty(max(1, capacity), np.uint64)
        cs, keep = c_scene if c_scene is not None else scene.c_struct()
        p = _abi.make_params(resolution, layout, gaussian_std, max_gaussians, flags)
        res = _abi.m2s_result()
        check(lib().m2s_convert_host(self.handle, C.byref(cs), C.byref(p), out.ctypes.data, capacity,
                                     keys.ctypes.data if want_keys else None, C.byref(res)),
              allow=(_abi.M2S_E_CAPACITY,))
        del keep
        rec = out[: res.written * stride].view(_abi.record_dtype(layout))
        return rec, (keys[: res.written] if want_keys else None), res

    # ---- outputs ----
    def ply_encode(self, ref96, count: int, fmt: int, scale_multiplier: float):
        """REF96 device tensor -> device tensor of .ply body rows."""
        torch = _torch()
        layout = _abi.PLY_FORMAT_LAYOUT.get(fmt, _abi.LAYOUT_PLY_STANDARD)
        rows = torch.empty(max(1, count) * _abi.STRIDES[layout], dtype=torch.uint8, device=ref96.device)
        check(lib().m2s_ply_encode(self.handle, ref96.data_ptr(), count, fmt, scale_multiplier, rows.data_ptr(), None))
        torch.cuda.synchronize(ref96.device)
        return rows[: count * _abi.STRIDES[layout]]

    # ---- .ply input (loadPlyFile) ----
    def ply_decode(self, rows, info: _abi.m2s_ply_info, out=None, count: int | None = None):
        """Decode .ply vertex rows already on the device (a torch uint8 tensor of count * info.row_stride bytes, any
        alignment) into REF96 records (m2s_ply_decode_enqueue on torch's current stream).  Returns the records as a torch
        uint8 device tensor of count * 96 bytes (out: optional caller-owned tensor of at least that size)."""
        torch = _torch()
        if count is None:
            count = rows.numel() // info.row_stride
        if out is None:
            out = torch.empty(max(1, count) * 96, dtype=torch.uint8, device=rows.device)
        check(lib().m2s_ply_decode_enqueue(self.handle, C.byref(info), rows.data_ptr(), count, out.data_ptr(),
                                           torch.cuda.current_stream(rows.device).cuda_stream))
        torch.cuda.synchronize(rows.device)
        return out[: count * 96]

    def ply_read(self, path: str, out=None):
        """SceneManager::loadPly's loadPlyFile on the GPU (m2s_ply_read): returns (records, count, has_pbr), records a
        torch uint8 device tensor of count * 96 bytes (REF96).  out: optional caller-owned device tensor; M2SError with
        M2S_E_CAPACITY when it holds fewer than count records."""
        torch = _torch()
        info = _abi.m2s_ply_info()
        check(lib().m2s_ply_read(self.handle, path.encode(), None, 0, C.byref(info)))
        n = int(info.vertex_count)
        if out is None:
            out = torch.empty(max(1, n) * 96, dtype=torch.uint8, device=torch.device("cuda", self.device))
        torch.cuda.synchronize(out.device)   # the buffer torch hands out is idle before the context stream writes it
        check(lib().m2s_ply_read(self.handle, path.encode(), out.data_ptr(), out.numel() // 96, C.byref(info)))
        return out[: n * 96], n, bool(info.has_pbr)

    def ply_read_sh(self, path: str, out=None, sh=None):
        """ply_read that also loads the SH rest coefficients (m2s_ply_read_sh): returns (records, sh, count, has_pbr,
        sh_degree); sh is a (count, M2S_SH_FLOATS(sh_degree)) float32 device tensor, coefficient-major with zero padding,
        or None for a file of degree 0.  out / sh: optional caller-owned device tensors (sh float32, at least count *
        M2S_SH_FLOATS(sh_degree) values); M2SError with M2S_E_CAPACITY when either holds fewer than count gaussians."""
        torch = _torch()
        info = _abi.m2s_ply_info()
        check(lib().m2s_ply_read_sh(self.handle, path.encode(), None, None, 0, C.byref(info)))
        n, deg = int(info.vertex_count), int(info.sh_degree)
        nf = _abi.SH_FLOATS[deg]
        dev = torch.device("cuda", self.device)
        if out is None:
            out = torch.empty(max(1, n) * 96, dtype=torch.uint8, device=dev)
        if nf and sh is None:
            sh = torch.empty(max(1, n) * nf, dtype=torch.float32, device=dev)
        cap = out.numel() // 96
        if nf:
            if sh.dtype != torch.float32 or not sh.is_contiguous():
                raise ValueError("sh must be a contiguous float32 device tensor")
            cap = min(cap, sh.numel() // nf)
        torch.cuda.synchronize(out.device)   # the buffers torch hands out are idle before the context stream writes them
        check(lib().m2s_ply_read_sh(self.handle, path.encode(), out.data_ptr(), sh.data_ptr() if nf else None, cap, C.byref(info)))
        return out[: n * 96], (sh.reshape(-1)[: n * nf].view(n, nf) if nf else None), n, bool(info.has_pbr), deg

    def ply_h2d_bytes(self) -> int:
        return int(lib().m2s_ply_h2d_bytes(self.handle))

    def convert_file(self, glb_path: str, resolution: int, ply_path: str, gaussian_std: float = 0.65, fmt: int = 0):
        res = _abi.m2s_result()
        check(lib().m2s_convert_file(self.handle, glb_path.encode(), resolution, gaussian_std, fmt, ply_path.encode(),
                                     C.byref(res)), allow=(_abi.M2S_E_CAPACITY,))
        return res


def depth_sort_tile() -> int:
    """Keys per tile of a depth-sort pass: the value the kernels use (m2s_debug_sort_tile, kept out of m2s.h)."""
    fn = lib().m2s_debug_sort_tile
    fn.restype = C.c_uint32
    fn.argtypes = []
    return int(fn())


def ply_header(fmt: int, count: int) -> bytes:
    buf = C.create_string_buffer(8192)
    n = lib().m2s_ply_header(fmt, count, buf, 8192)
    return buf.raw[:n]


def ply_parse_header(data: bytes, file_size: int | None = None) -> _abi.m2s_ply_info:
    """m2s_ply_parse_header on the first bytes of a .ply file (file_size: the whole file's size, default len(data)).
    Raises M2SError (M2S_E_FORMAT with the cause) for a file the loader does not take."""
    info = _abi.m2s_ply_info()
    buf = C.create_string_buffer(bytes(data), len(data))
    check(lib().m2s_ply_parse_header(buf, len(data), len(data) if file_size is None else int(file_size), C.byref(info)))
    return info


def ply_parse_file(path: str) -> _abi.m2s_ply_info:
    """ply_parse_header on a file: its first 1 MB and its size."""
    import os
    with open(path, "rb") as f:
        head = f.read(1 << 20)
    return ply_parse_header(head, os.path.getsize(path))


def write_3dgs_ply(path: str, params) -> None:
    """PACKED56 gaussians (an (n, 14) float32 array or tensor: xyz, quaternion wxyz, log-scale, SH0, opacity logit) as a
    standard 3DGS .ply: the header of m2s_ply_header format 0 (LAYOUT_PLY_STANDARD), the fields as they are, zero normals
    and f_rest."""
    a = params.detach().cpu().numpy() if hasattr(params, "detach") else np.asarray(params)
    a = np.asarray(a, np.float32).reshape(-1, 14)
    rows = np.zeros(len(a), _abi.record_dtype(_abi.LAYOUT_PLY_STANDARD))
    rows["xyz"], rows["f_dc"], rows["opacity"], rows["scale"], rows["rot"] = a[:, 0:3], a[:, 10:13], a[:, 13], a[:, 7:10], a[:, 3:7]
    with open(path, "wb") as f:
        f.write(ply_header(0, len(a)))
        f.write(rows.tobytes())


def ply_write(path: str, ref96: np.ndarray, fmt: int, scale_multiplier: float) -> None:
    a = np.ascontiguousarray(ref96)
    count = a.nbytes // 96
    check(lib().m2s_ply_write(path.encode(), a.ctypes.data, count, fmt, scale_multiplier))


# ---------------------------------------------------------------------------------------------
# reference-shaped objects
# ---------------------------------------------------------------------------------------------
class Gs3dState:
    """m2s_3dgs_state: what one forward pass of Context.render_3dgs_grad keeps for its backward pass."""

    def __init__(self, ctx: Context):
        h = C.c_void_p(0)
        check(lib().m2s_3dgs_state_create(ctx.handle, C.byref(h)))
        self.handle = h.value
        self.generation = 0   # counts the forward passes; a backward checks that its own is still the one held

    def free(self):
        if getattr(self, "handle", 0):
            lib().m2s_3dgs_state_destroy(self.handle)
            self.handle = 0

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.free()


_CUDA_STREAM_LEGACY = 1   # cudaStreamLegacy: the default stream torch's handle 0 stands for


def _render_3dgs_grad_class():
    torch = _torch()

    class Render3dgsGrad(torch.autograd.Function):
        @staticmethod
        def forward(fctx, params, ctx, state, p, max_pairs):
            assert params.dtype == torch.float32 and params.is_cuda and params.dim() == 2 and params.shape[1] == 14, params.shape
            params = params.detach().contiguous()
            dev = params.device
            count = params.shape[0]
            img = torch.empty(p.height * p.width * 4, dtype=torch.float32, device=dev)
            _binned_pass(dev, max_pairs, count,
                         lambda pairs: lib().m2s_3dgs_render_grad(ctx.handle, state.handle, params.data_ptr(), count, C.byref(p),
                                                                  img.data_ptr(), pairs),
                         lambda *budget: lib().m2s_3dgs_render_grad_enqueue(ctx.handle, state.handle, params.data_ptr(), count,
                                                                            C.byref(p), img.data_ptr(), *budget))
            state.generation += 1
            fctx.save_for_backward(params)   # torch's version counter: an in-place change before the backward raises
            fctx.saved = (ctx, state, p, state.generation)
            return img.view(p.height, p.width, 4)

        @staticmethod
        def backward(fctx, grad_img):
            (params,) = fctx.saved_tensors
            ctx, state, p, gen = fctx.saved
            if state.generation != gen:
                raise RuntimeError("render_3dgs_grad: the state has since held another forward pass; use one state per view")
            g = grad_img.detach().to(torch.float32).contiguous()
            grad = torch.empty_like(params)
            # torch's current stream; its default stream has handle 0, which the C ABI reads as "the context's stream" (not
            # ordered with torch's work), so that one is named as cudaStreamLegacy (0x1)
            stream = torch.cuda.current_stream(params.device).cuda_stream or _CUDA_STREAM_LEGACY
            check(lib().m2s_3dgs_backward_enqueue(ctx.handle, state.handle, params.data_ptr(), params.shape[0], C.byref(p), g.data_ptr(),
                                                  grad.data_ptr(), stream))
            return grad, None, None, None, None

    return Render3dgsGrad


class _LazyFunction:
    """The autograd Function, made on first use (torch is imported lazily)."""
    fn = None

    def apply(self, *args):
        if _LazyFunction.fn is None:
            _LazyFunction.fn = _render_3dgs_grad_class()
        return _LazyFunction.fn.apply(*args)


_Render3dgsGrad = _LazyFunction()


class RenderContext:
    """The fields of struct RenderContext (RenderContext.hpp:28-124) the conversion path touches."""

    def __init__(self, device: int = 0):
        self.ctx = Context(device)
        self.resolutionTarget = 520          # ImGuiUI.cpp:512 at the default quality 0.5
        self.gaussianStd = 0.65              # main.cpp:26
        self.scene: _abi.Scene | None = None       # dataMeshAndGlMesh (CPU side)
        self.deviceScene: DeviceScene | None = None  # ... (GPU side) + meshToTextureData
        self.gaussianBuffer = None           # SSBO: torch.uint8 device tensor of GaussianDataSSBO records
        self.numberOfGaussians = 0           # may exceed the buffer capacity (ConversionPass.cpp:56-59)
        self.lastResult: ConvertOutput | None = None
        self.format = 0                      # u_format: 0 the conversion's records, 1 a loaded .ply (RenderContext.hpp)
        self.plyHasPbr = False               # format 1: the .ply carries normals and metallic / roughness
        self.shCoefficients = None           # format 1 loaded withSh: (n, 12 | 24 | 48) float32 device tensor (beyond the reference)
        self.shDegree = 0                    # ... its degree (0: no view-dependent colour)

    def viewLayout(self) -> int:
        """The `layout` the viewer passes (prepass, shadow_map) take for gaussianBuffer."""
        if self.format == 1:
            return _abi.VIEW_PLY_PBR if self.plyHasPbr else _abi.VIEW_PLY
        return _abi.LAYOUT_REF96


class SceneManager:
    def __init__(self, renderContext: RenderContext):
        self.renderContext = renderContext

    def setScene(self, scene: _abi.Scene) -> bool:
        rc = self.renderContext
        if rc.deviceScene is not None:
            rc.deviceScene.free()
        rc.scene = scene
        rc.deviceScene = rc.ctx.upload(scene)
        return True

    def loadModel(self, filePath: str, parentFolder: str = "") -> bool:
        """SceneManager::loadModel (SceneManager.cpp:22-35): parse .glb, bboxes, textures -> GPU."""
        from .gltf import load_glb  # noqa: WPS433
        try:
            return self.setScene(load_glb(filePath))
        except (OSError, ValueError) as e:  # the reference prints and returns false
            print(f"Failed to parse GLTF file: {filePath}: {e}")
            return False

    def loadPly(self, filePath: str, withSh: bool = False) -> bool:
        """SceneManager::loadPly (SceneManager.cpp:37-47) + parsers::loadPlyFile: the file's gaussians become
        gaussianBuffer (REF96 on the device), format 1, plyHasPbr from the file.  withSh (beyond the reference): also
        load the SH rest coefficients into shCoefficients / shDegree (prepass(sh=...)); without it they are None / 0, as
        the reference skips them.  Deviation: a file the loader does not take returns False and leaves the previous
        gaussians in place (the reference prints the error and returns true)."""
        rc = self.renderContext
        try:
            ply_parse_file(filePath)   # header and size checked on the host before anything reaches the device
            if withSh:
                records, sh, n, has_pbr, degree = rc.ctx.ply_read_sh(filePath)
            else:
                (records, n, has_pbr), sh, degree = rc.ctx.ply_read(filePath), None, 0
        except (OSError, M2SError) as e:
            print(f"Error loading PLY file: {filePath}: {e}")
            return False
        rc.gaussianBuffer, rc.numberOfGaussians, rc.format, rc.plyHasPbr = records, n, 1, has_pbr
        rc.shCoefficients, rc.shDegree = sh, degree
        return True

    def exportPly(self, outputFile: str, exportFormat: int = 0) -> None:
        """SceneManager::exportPly (SceneManager.cpp:651-678): read back, scale by std/R, write."""
        rc = self.renderContext
        out = rc.lastResult
        if out is None:
            raise RuntimeError("exportPly before ConversionPass.execute")
        mult = np.float32(rc.gaussianStd) / np.float32(rc.resolutionTarget)
        ply_write(outputFile, out.numpy(), exportFormat, float(mult))


class ConversionPass:
    """IRenderPass for the conversion (RenderPass.hpp:10-28, ConversionPass.cpp:9-68)."""

    def __init__(self):
        self._enabled = False

    def isEnabled(self) -> bool:
        return self._enabled

    def setIsEnabled(self, isPassEnabled: bool) -> None:
        self._enabled = bool(isPassEnabled)

    def execute(self, renderContext: RenderContext) -> None:
        rc = renderContext
        if rc.deviceScene is None:
            raise RuntimeError("ConversionPass.execute: no model loaded")
        out = rc.ctx.convert(rc.deviceScene, rc.resolutionTarget, _abi.LAYOUT_REF96, rc.gaussianStd)
        rc.gaussianBuffer = out.data
        rc.numberOfGaussians = out.total
        rc.lastResult = out


__all__ = ["Context", "DeviceScene", "ConvertOutput", "RenderContext", "SceneManager", "ConversionPass", "depth_sort_tile",
           "ply_header", "ply_write", "ply_parse_header", "ply_parse_file", "M2SError"]
