"""ctypes mirror of include/m2s.h (structs, enums) and the host-side Scene container.

No compute here: this is the marshalling layer between numpy arrays and the C ABI.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass, field

import numpy as np

# ---- enums (include/m2s.h) ------------------------------------------------------------------
M2S_OK, M2S_E_INVALID, M2S_E_NOGPU, M2S_E_CUDA, M2S_E_CAPACITY, M2S_E_IO, M2S_E_FORMAT = range(7)
LAYOUT_REF96, LAYOUT_PACKED56, LAYOUT_PLY_STANDARD, LAYOUT_PLY_PBR, LAYOUT_PLY_COMPRESSED = range(5)
FLAG_NONE, FLAG_UNCAPPED = 0, 1
FLOATS_PER_TRIANGLE = 36
MAX_MIP_LEVEL = 4
REFERENCE_MAX_GAUSSIANS = 7_000_000
STRIDES = {LAYOUT_REF96: 96, LAYOUT_PACKED56: 56, LAYOUT_PLY_STANDARD: 248, LAYOUT_PLY_PBR: 76,
           LAYOUT_PLY_COMPRESSED: 48}
# which .ply format (savePlyVector FORMAT, parsers.cpp:631-651) a row layout corresponds to
PLY_FORMAT_LAYOUT = {0: LAYOUT_PLY_STANDARD, 1: LAYOUT_PLY_PBR, 2: LAYOUT_PLY_COMPRESSED}
# viewer-pass input: REF96 records as m2s_ply_read loads them (u_format 1, u_plyHasPbr 0 / 1)
VIEW_PLY, VIEW_PLY_PBR = 16, 17
# m2s_ply_info.offset: the properties loadPlyFile reads, in this order
PLY_PROPS = ("x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2", "metallicFactor", "roughnessFactor", "opacity",
             "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3")
PLY_MAX_STRIDE = 4096
# SH rest coefficients of a loaded .ply (m2s_ply_info.sh_degree): floats per gaussian of an SH buffer by degree
SH_REST_MAX = 45
SH_FLOATS = {0: 0, 1: 12, 2: 24, 3: 48}
# m2s_debug_codec_eval function ids (m2s_codec.cu; not in m2s.h)
CODEC_SH0, CODEC_LOGIT, CODEC_LOG_SCALE, CODEC_EXPF, CODEC_SIGMOID = range(5)


class m2s_ply_info(C.Structure):
    """include/m2s.h: what m2s_ply_parse_header reads from a .ply header."""
    _fields_ = [("vertex_count", C.c_uint64), ("body_offset", C.c_uint64), ("row_stride", C.c_uint32), ("has_pbr", C.c_uint32),
                ("offset", C.c_int32 * len(PLY_PROPS)), ("sh_degree", C.c_uint32), ("f_rest", C.c_int32 * SH_REST_MAX)]

    def offsets(self) -> dict:
        """{property name: byte offset in the row} of the properties present."""
        return {n: int(o) for n, o in zip(PLY_PROPS, self.offset) if o >= 0}


class m2s_texture(C.Structure):
    _fields_ = [("rgba", C.c_void_p), ("width", C.c_uint32), ("height", C.c_uint32)]


class m2s_primitive(C.Structure):
    _fields_ = [("first_triangle", C.c_uint64), ("triangle_count", C.c_uint64),
                ("bbox_min", C.c_float * 3), ("bbox_max", C.c_float * 3),
                ("base_color_factor", C.c_float * 4),
                ("albedo_texture", C.c_int32), ("normal_texture", C.c_int32),
                ("metallic_roughness_texture", C.c_int32), ("reserved", C.c_int32)]


class m2s_scene(C.Structure):
    _fields_ = [("triangles", C.c_void_p), ("triangle_count", C.c_uint64),
                ("primitives", C.POINTER(m2s_primitive)), ("primitive_count", C.c_uint32),
                ("textures", C.POINTER(m2s_texture)), ("texture_count", C.c_uint32)]


class m2s_params(C.Structure):
    _fields_ = [("resolution", C.c_uint32), ("gaussian_std", C.c_float),
                ("max_gaussians", C.c_uint64), ("layout", C.c_uint32), ("flags", C.c_uint32),
                ("first_triangle", C.c_uint64), ("triangle_count", C.c_uint64),
                ("row_begin", C.c_uint32), ("row_end", C.c_uint32)]


class m2s_result(C.Structure):
    _fields_ = [("total", C.c_uint64), ("written", C.c_uint64), ("cap", C.c_uint64),
                ("device_ms", C.c_float)]


class m2s_convert_plan(C.Structure):
    """ConvertPlan (m2s_convert.cu), filled by m2s_debug_convert_plan: the launch a conversion makes and its route."""
    _fields_ = [(n, C.c_uint64) for n in ("grid", "raster_warps", "unit_tris", "n_units", "item_max", "flush_frags",
                                          "queue_cap", "cap", "multi_round", "direct_ok", "claim_late", "direct_max",
                                          "pair_first", "single_launch")]


MAX_PEERS = 8


class m2s_prepass_params(C.Structure):
    """include/m2s.h: the uniforms of GaussiansPrepass::execute; matrices column-major (glm::mat4)."""
    _fields_ = [("world_to_view", C.c_float * 16), ("view_to_clip", C.c_float * 16), ("model_to_world", C.c_float * 16),
                ("resolution", C.c_float * 2), ("near_far", C.c_float * 2), ("std_dev", C.c_float), ("render_mode", C.c_uint32),
                ("layout", C.c_uint32), ("reserved", C.c_uint32)]


QUAD_BYTES = 96


class m2s_gbuffer(C.Structure):
    """include/m2s.h: the five G-buffer targets of GaussianSplattingPass (device pointers, NULL = not drawn)."""
    _fields_ = [("position", C.c_void_p), ("normal", C.c_void_p), ("albedo", C.c_void_p), ("depth", C.c_void_p),
                ("metallic_roughness", C.c_void_p)]


class m2s_splat_params(C.Structure):
    _fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("render_mode", C.c_uint32)]


class m2s_shadow_params(C.Structure):
    """include/m2s.h: the uniforms of GaussianShadowPass::execute; model_to_world column-major (glm::mat4)."""
    _fields_ = [("model_to_world", C.c_float * 16), ("light_position", C.c_float * 3), ("near_far", C.c_float * 2),
                ("resolution", C.c_float * 2), ("std_dev", C.c_float), ("layout", C.c_uint32), ("size", C.c_uint32)]


class m2s_light_params(C.Structure):
    """include/m2s.h: the uniforms of GaussianRelightingPass::execute."""
    _fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("render_mode", C.c_uint32), ("light_position", C.c_float * 3),
                ("light_color", C.c_float * 3), ("light_intensity", C.c_float), ("cam_pos", C.c_float * 3), ("far_plane", C.c_float),
                ("shadow_size", C.c_uint32)]


LIGHT_RECORD_BYTES = 32


def make_shadow_params(model_to_world, light_position, near_far, resolution, std_dev: float, layout: int, size: int = 1024):
    p = m2s_shadow_params()
    p.model_to_world = (C.c_float * 16)(*[float(v) for v in np.asarray(model_to_world, np.float32).ravel()])
    p.light_position = (C.c_float * 3)(*[float(v) for v in light_position])
    p.near_far = (C.c_float * 2)(float(near_far[0]), float(near_far[1]))
    p.resolution = (C.c_float * 2)(float(resolution[0]), float(resolution[1]))
    p.std_dev, p.layout, p.size = float(std_dev), int(layout), int(size)
    return p


def make_light_params(width: int, height: int, render_mode: int, light_position=(0.0, 0.0, 0.0), light_color=(1.0, 1.0, 1.0),
                      light_intensity: float = 1.0, cam_pos=(0.0, 0.0, 0.0), far_plane: float = 100.0, shadow_size: int = 1024):
    p = m2s_light_params()
    p.width, p.height, p.render_mode = int(width), int(height), int(render_mode)
    p.light_position = (C.c_float * 3)(*[float(v) for v in light_position])
    p.light_color = (C.c_float * 3)(*[float(v) for v in light_color])
    p.cam_pos = (C.c_float * 3)(*[float(v) for v in cam_pos])
    p.light_intensity, p.far_plane, p.shadow_size = float(light_intensity), float(far_plane), int(shadow_size)
    return p


# G-buffer attachments in order (renderer.cpp:325-379): name, element dtype (float16 bits or uint8)
GBUFFER_TARGETS = (("position", np.float16), ("normal", np.float16), ("albedo", np.uint8), ("depth", np.float16),
                   ("metallic_roughness", np.uint8))


def make_prepass_params(world_to_view, view_to_clip, model_to_world, resolution, near_far, std_dev: float, render_mode: int, layout: int):
    p = m2s_prepass_params()
    for name, m in (("world_to_view", world_to_view), ("view_to_clip", view_to_clip), ("model_to_world", model_to_world)):
        setattr(p, name, (C.c_float * 16)(*[float(v) for v in np.asarray(m, np.float32).ravel()]))
    p.resolution = (C.c_float * 2)(float(resolution[0]), float(resolution[1]))
    p.near_far = (C.c_float * 2)(float(near_far[0]), float(near_far[1]))
    p.std_dev, p.render_mode, p.layout, p.reserved = float(std_dev), int(render_mode), int(layout), 0
    return p


class m2s_mesh_depth_params(C.Structure):
    """include/m2s.h: the uniforms of DepthPrepass::execute; matrices column-major (glm::mat4)."""
    _fields_ = [("world_to_view", C.c_float * 16), ("view_to_clip", C.c_float * 16), ("model_to_world", C.c_float * 16),
                ("width", C.c_uint32), ("height", C.c_uint32)]


def make_mesh_depth_params(world_to_view, view_to_clip, model_to_world, width: int, height: int):
    p = m2s_mesh_depth_params()
    for name, m in (("world_to_view", world_to_view), ("view_to_clip", view_to_clip), ("model_to_world", model_to_world)):
        setattr(p, name, (C.c_float * 16)(*[float(v) for v in np.asarray(m, np.float32).ravel()]))
    p.width, p.height = int(width), int(height)
    return p


class m2s_mesh_render_params(C.Structure):
    """include/m2s.h: the uniforms of MeshRenderPass::execute; matrices column-major (glm::mat4)."""
    _fields_ = [("world_to_view", C.c_float * 16), ("view_to_clip", C.c_float * 16), ("model_to_world", C.c_float * 16),
                ("near_far", C.c_float * 2), ("width", C.c_uint32), ("height", C.c_uint32), ("render_mode", C.c_uint32)]


def make_mesh_render_params(world_to_view, view_to_clip, model_to_world, width: int, height: int, near_far, render_mode: int = 0):
    p = m2s_mesh_render_params()
    for name, m in (("world_to_view", world_to_view), ("view_to_clip", view_to_clip), ("model_to_world", model_to_world)):
        setattr(p, name, (C.c_float * 16)(*[float(v) for v in np.asarray(m, np.float32).ravel()]))
    p.near_far = (C.c_float * 2)(float(near_far[0]), float(near_far[1]))
    p.width, p.height, p.render_mode = int(width), int(height), int(render_mode)
    return p


class m2s_3dgs_params(C.Structure):
    """include/m2s.h: the camera, image and records of the standard 3DGS render; matrices column-major (glm::mat4)."""
    _fields_ = [("world_to_view", C.c_float * 16), ("view_to_clip", C.c_float * 16), ("model_to_world", C.c_float * 16),
                ("width", C.c_uint32), ("height", C.c_uint32), ("near", C.c_float), ("std_dev", C.c_float), ("scale_modifier", C.c_float),
                ("background", C.c_float * 3), ("layout", C.c_uint32), ("reserved", C.c_uint32)]


GS3D_SPLAT_FLOATS = 12   # the preprocess kernel's splat record (m2s_debug_3dgs_preprocess): 48 B
GS3D_CULLED = 0xFFFFFFFF  # the depth key of a culled record


def make_3dgs_params(world_to_view, view_to_clip, model_to_world, width: int, height: int, near: float, std_dev: float,
                     scale_modifier: float, background, layout: int):
    p = m2s_3dgs_params()
    for name, m in (("world_to_view", world_to_view), ("view_to_clip", view_to_clip), ("model_to_world", model_to_world)):
        setattr(p, name, (C.c_float * 16)(*[float(v) for v in np.asarray(m, np.float32).ravel()]))
    p.width, p.height = int(width), int(height)
    p.near, p.std_dev, p.scale_modifier = float(near), float(std_dev), float(scale_modifier)
    p.background = (C.c_float * 3)(*[float(v) for v in background])
    p.layout, p.reserved = int(layout), 0
    return p


class m2s_compare_params(C.Structure):
    _fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("cover_min", C.c_uint32)]


class m2s_compare_result(C.Structure):
    """include/m2s.h: the totals of m2s_image_compare."""
    _fields_ = [("windows", C.c_uint64), ("covered_windows", C.c_uint64), ("pixels_both", C.c_uint64), ("pixels_a_only", C.c_uint64),
                ("pixels_b_only", C.c_uint64), ("sq_err", C.c_uint64 * 3), ("sq_err_covered", C.c_uint64 * 3), ("ssim", C.c_double * 3),
                ("ssim_covered", C.c_double * 3)]


def psnr(sq_err_sum: int, samples: int) -> float:
    """10 log10(255^2 samples / sq_err_sum), samples = 3 N channel values; +inf for no error, nan for no samples."""
    if samples == 0:
        return float("nan")
    return float("inf") if sq_err_sum == 0 else 10.0 * math.log10(255.0 * 255.0 * samples / sq_err_sum)


def compare_result_dict(r: m2s_compare_result, pixels: int) -> dict:
    """The totals of an m2s_compare_result as a dict, plus psnr, ssim (sum over channels / 3 windows) and the covered
    forms (nan with nothing covered)."""
    d = {n: int(getattr(r, n)) for n in ("windows", "covered_windows", "pixels_both", "pixels_a_only", "pixels_b_only")}
    for n in ("sq_err", "sq_err_covered"):
        d[n] = [int(v) for v in getattr(r, n)]
    for n in ("ssim_sum", "ssim_covered_sum"):
        d[n] = [float(v) for v in getattr(r, n.replace("_sum", ""))]
    covered = d["pixels_both"] + d["pixels_a_only"] + d["pixels_b_only"]
    d["psnr"] = psnr(sum(d["sq_err"]), 3 * pixels)
    d["psnr_covered"] = psnr(sum(d["sq_err_covered"]), 3 * covered)
    d["ssim"] = math.fsum(d["ssim_sum"]) / (3 * d["windows"])
    d["ssim_covered"] = math.fsum(d["ssim_covered_sum"]) / (3 * d["covered_windows"]) if d["covered_windows"] else float("nan")
    return d


class m2s_peers(C.Structure):
    _fields_ = [("world", C.c_uint32), ("rank", C.c_uint32), ("out", C.c_void_p * MAX_PEERS), ("xch", C.c_void_p * MAX_PEERS)]


def make_params(resolution: int, layout: int = LAYOUT_REF96, gaussian_std: float = 0.65,
                max_gaussians: int = 0, flags: int = 0, first_triangle: int = 0,
                triangle_count: int = 0, row_begin: int = 0, row_end: int = 0) -> m2s_params:
    return m2s_params(int(resolution), float(gaussian_std), int(max_gaussians), int(layout),
                      int(flags), int(first_triangle), int(triangle_count), int(row_begin), int(row_end))


def reference_capacity(resolution: int, primitive_count: int) -> int:
    """min(6 R^2 meshCount, 7e6): ConversionPass.cpp:21-24."""
    return min(6 * resolution * resolution * max(1, primitive_count), REFERENCE_MAX_GAUSSIANS)


@dataclass
class Primitive:
    """One glTF primitive == one utils::Mesh == one draw call of the reference."""
    first_triangle: int
    triangle_count: int
    base_color_factor: tuple = (1.0, 1.0, 1.0, 1.0)
    albedo_texture: int = -1
    normal_texture: int = -1
    metallic_roughness_texture: int = -1
    bbox_min: tuple = (0.0, 0.0, 0.0)
    bbox_max: tuple = (0.0, 0.0, 0.0)
    name: str = "mesh"


@dataclass
class Scene:
    """Host-side scene: what SceneManager::loadModel leaves in RenderContext, minus GL handles.

    triangles: float32 (T, 36) — 3 x {position xyz, normal xyz, tangent xyzw, uv}, world space
    textures:  list of uint8 (H, W, 4), row 0 first
    """
    triangles: np.ndarray
    primitives: list = field(default_factory=list)
    textures: list = field(default_factory=list)

    def __post_init__(self):
        t = np.ascontiguousarray(self.triangles, dtype=np.float32)
        if t.ndim != 2 or t.shape[1] != FLOATS_PER_TRIANGLE:
            t = t.reshape(-1, FLOATS_PER_TRIANGLE)
        self.triangles = t
        self.textures = [np.ascontiguousarray(x, dtype=np.uint8) for x in self.textures]
        for x in self.textures:
            if x.ndim != 3 or x.shape[2] != 4:
                raise ValueError("textures must be (H, W, 4) uint8")
        if not self.primitives:
            self.primitives = [Primitive(0, len(t))]

    @property
    def triangle_count(self) -> int:
        return int(self.triangles.shape[0])

    def compute_bboxes(self, cumulative: bool = True) -> None:
        """Reference rule (SceneManager.cpp:476-477,514-520,527): primitive k gets the union box
        of primitives 0..k when cumulative (the reference's behaviour)."""
        mn = np.full(3, np.finfo(np.float32).max, np.float32)
        mx = -mn
        pos = self.triangles.reshape(-1, 3, 12)[:, :, 0:3]
        for p in self.primitives:
            if not cumulative:
                mn = np.full(3, np.finfo(np.float32).max, np.float32)
                mx = -mn
            sl = pos[p.first_triangle:p.first_triangle + p.triangle_count].reshape(-1, 3)
            if len(sl):
                mn = np.minimum(mn, sl.min(axis=0))
                mx = np.maximum(mx, sl.max(axis=0))
            p.bbox_min = tuple(float(v) for v in mn)
            p.bbox_max = tuple(float(v) for v in mx)

    def c_struct(self):
        """Returns (m2s_scene, keepalive) — keep `keepalive` referenced while the struct is used."""
        prims = (m2s_primitive * max(1, len(self.primitives)))()
        for i, p in enumerate(self.primitives):
            prims[i].first_triangle = p.first_triangle
            prims[i].triangle_count = p.triangle_count
            prims[i].bbox_min = (C.c_float * 3)(*p.bbox_min)
            prims[i].bbox_max = (C.c_float * 3)(*p.bbox_max)
            prims[i].base_color_factor = (C.c_float * 4)(*p.base_color_factor)
            prims[i].albedo_texture = p.albedo_texture
            prims[i].normal_texture = p.normal_texture
            prims[i].metallic_roughness_texture = p.metallic_roughness_texture
        texs = (m2s_texture * max(1, len(self.textures)))()
        for i, t in enumerate(self.textures):
            texs[i].rgba = t.ctypes.data
            texs[i].width = t.shape[1]
            texs[i].height = t.shape[0]
        s = m2s_scene()
        s.triangles = self.triangles.ctypes.data
        s.triangle_count = self.triangle_count
        s.primitives = prims
        s.primitive_count = len(self.primitives)
        s.textures = texs
        s.texture_count = len(self.textures)
        return s, (prims, texs, self.triangles, self.textures)

    def texture_bytes(self) -> int:
        return int(sum(t.nbytes for t in self.textures))


def record_dtype(layout: int) -> np.dtype:
    """numpy view of one output record."""
    if layout == LAYOUT_REF96:
        return np.dtype([("position", "<f4", 4), ("color", "<f4", 4), ("scale", "<f4", 4),
                         ("normal", "<f4", 4), ("rotation", "<f4", 4), ("pbr", "<f4", 4)])
    if layout == LAYOUT_PACKED56:
        return np.dtype([("xyz", "<f4", 3), ("rot", "<f4", 4), ("log_scale", "<f4", 3),
                         ("sh0", "<f4", 3), ("opacity", "<f4")])
    if layout == LAYOUT_PLY_STANDARD:
        return np.dtype([("xyz", "<f4", 3), ("normal", "<f4", 3), ("f_dc", "<f4", 3),
                         ("f_rest", "<f4", 45), ("opacity", "<f4"), ("scale", "<f4", 3),
                         ("rot", "<f4", 4)])
    if layout == LAYOUT_PLY_PBR:
        return np.dtype([("xyz", "<f4", 3), ("normal", "<f4", 3), ("f_dc", "<f4", 3),
                         ("metallic", "<f4"), ("roughness", "<f4"), ("opacity", "<f4"),
                         ("scale", "<f4", 3), ("rot", "<f4", 4)])
    if layout == LAYOUT_PLY_COMPRESSED:
        return np.dtype([("xyz", "<f4", 3), ("rgba", "u1", 4), ("rot", "<f4", 4),
                         ("scale", "<f4", 3), ("octa", "u1", 2), ("roughness", "u1"),
                         ("metallic", "u1")])
    raise ValueError(f"unknown layout {layout}")
