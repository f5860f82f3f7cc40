"""ctypes binding of the native scene front end (include/vello_b200_scene.h, vello_b200/csrc/vb_scene.cpp).

`NativeScene` has the call surface of `vello_b200.encoding.Scene` (= `vello::Scene`, vello/src/scene.rs) and takes the same
Python value objects; every call goes straight into libvello_b200.so. `resolve()` returns the same `Packed` the Python
encoder produces -- byte for byte, which tests/test_scene_native.py asserts on every test scene."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from . import shapes as _shapes
from .encoding import Color, Gradient, Image, Layout, Packed, Stroke
from .renderer import _Layout, load_library
from .shapes import Affine


class _Path(C.Structure):
    _fields_ = [("verbs", C.c_void_p), ("n_verbs", C.c_uint32), ("coords", C.c_void_p)]


class _Color(C.Structure):
    _fields_ = [("r", C.c_float), ("g", C.c_float), ("b", C.c_float), ("a", C.c_float)]


class _Stop(C.Structure):
    _fields_ = [("offset", C.c_float), ("color", _Color)]


class _Image(C.Structure):
    _fields_ = [("pixels", C.c_void_p), ("width", C.c_uint32), ("height", C.c_uint32), ("format", C.c_uint32), ("alpha_type", C.c_uint32),
                ("quality", C.c_uint32), ("x_extend", C.c_uint32), ("y_extend", C.c_uint32), ("alpha", C.c_float)]


class _Brush(C.Structure):
    _fields_ = [("kind", C.c_uint32), ("color", _Color), ("geom", C.c_double * 6), ("stops", C.c_void_p), ("n_stops", C.c_uint32),
                ("extend", C.c_uint32), ("premul_interp", C.c_uint32), ("image", C.c_void_p)]


class _Stroke(C.Structure):
    _fields_ = [("width", C.c_double), ("join", C.c_uint32), ("start_cap", C.c_uint32), ("end_cap", C.c_uint32), ("miter_limit", C.c_double),
                ("dash_pattern", C.c_void_p), ("n_dashes", C.c_uint32), ("dash_offset", C.c_double)]


class _Packed(C.Structure):
    _fields_ = [("scene", C.c_void_p), ("scene_len", C.c_size_t), ("layout", _Layout), ("ramps", C.c_void_p), ("ramp_w", C.c_uint32),
                ("ramp_h", C.c_uint32), ("atlas", C.c_void_p), ("atlas_w", C.c_uint32), ("atlas_h", C.c_uint32)]


PATHBUF_SYMBOLS = ["vb_pathbuf_new", "vb_pathbuf_free", "vb_pathbuf_clear", "vb_pathbuf_move_to", "vb_pathbuf_line_to", "vb_pathbuf_quad_to",
                   "vb_pathbuf_curve_to", "vb_pathbuf_close", "vb_pathbuf_rect", "vb_pathbuf_line", "vb_pathbuf_circle", "vb_pathbuf_rounded_rect",
                   "vb_pathbuf_ellipse", "vb_pathbuf_arc",
                   "vb_pathbuf_svg", "vb_pathbuf_view"]
SCENE_SYMBOLS = ["vb_scene_new", "vb_scene_free", "vb_scene_reset", "vb_scene_fill", "vb_scene_stroke", "vb_scene_push_layer",
                 "vb_scene_push_luminance_mask_layer", "vb_scene_push_clip_layer", "vb_scene_pop_layer", "vb_scene_draw_image",
                 "vb_scene_draw_blurred_rounded_rect", "vb_scene_draw_blurred_rounded_rect_in", "vb_scene_append", "vb_scene_batch", "vb_scene_resolve", "vb_render_scene", "vb_scene_upload_device", "vb_path_dash",
                 "vb_register_texture", "vb_unregister_texture", "vb_scene_n_draw_objects", "vb_scene_upload_fragment",
                 "vb_scene_n_points", "vb_scene_n_stops", "vb_scene_n_transforms"]

_bound = False


def _lib():
    global _bound
    lib = load_library()
    if not _bound:
        vp = C.c_void_p
        lib.vb_scene_new.restype = vp
        lib.vb_scene_free.argtypes = [vp]
        lib.vb_scene_reset.argtypes = [vp]
        lib.vb_scene_n_draw_objects.restype = C.c_uint32
        lib.vb_scene_n_draw_objects.argtypes = [vp]
        lib.vb_scene_n_points.restype = C.c_uint32
        lib.vb_scene_n_points.argtypes = [vp]
        lib.vb_scene_n_stops.restype = C.c_uint32
        lib.vb_scene_n_stops.argtypes = [vp]
        lib.vb_scene_n_transforms.restype = C.c_uint32
        lib.vb_scene_n_transforms.argtypes = [vp]
        lib.vb_scene_fill.argtypes = [vp, C.c_uint32, vp, vp, vp, vp]
        lib.vb_scene_stroke.argtypes = [vp, vp, vp, vp, vp, vp]
        lib.vb_scene_push_layer.argtypes = [vp, C.c_uint32, vp, C.c_uint32, C.c_uint32, C.c_float, vp, vp]
        lib.vb_scene_push_luminance_mask_layer.argtypes = [vp, C.c_uint32, vp, C.c_float, vp, vp]
        lib.vb_scene_push_clip_layer.argtypes = [vp, C.c_uint32, vp, vp, vp]
        lib.vb_scene_pop_layer.argtypes = [vp]
        lib.vb_scene_draw_image.argtypes = [vp, vp, vp]
        lib.vb_scene_draw_blurred_rounded_rect.argtypes = [vp, vp, vp, _Color, C.c_double, C.c_double]
        lib.vb_scene_draw_blurred_rounded_rect_in.argtypes = [vp, vp, vp, vp, _Color, C.c_double, C.c_double]
        lib.vb_scene_append.argtypes = [vp, vp, vp]
        lib.vb_scene_batch.argtypes = [vp, vp, C.c_uint32, vp]
        lib.vb_scene_resolve.argtypes = [vp, vp]
        lib.vb_render_scene.argtypes = [vp, vp, vp, vp, C.c_uint32, vp]
        lib.vb_scene_upload_device.argtypes = [vp, vp, vp]
        lib.vb_scene_upload_fragment.argtypes = [vp, vp, vp]
        lib.vb_path_dash.argtypes = [vp, C.c_double, vp, C.c_uint32, vp]
        lib.vb_register_texture.argtypes = [vp, vp, C.c_uint32, C.c_uint32, C.c_size_t, C.POINTER(_Image)]
        lib.vb_unregister_texture.argtypes = [vp, C.POINTER(_Image)]
        d = C.c_double
        lib.vb_pathbuf_new.restype = vp
        lib.vb_pathbuf_free.argtypes = [vp]
        lib.vb_pathbuf_clear.argtypes = [vp]
        lib.vb_pathbuf_move_to.argtypes = [vp, d, d]
        lib.vb_pathbuf_line_to.argtypes = [vp, d, d]
        lib.vb_pathbuf_quad_to.argtypes = [vp, d, d, d, d]
        lib.vb_pathbuf_curve_to.argtypes = [vp, d, d, d, d, d, d]
        lib.vb_pathbuf_close.argtypes = [vp]
        lib.vb_pathbuf_rect.argtypes = [vp, d, d, d, d]
        lib.vb_pathbuf_line.argtypes = [vp, d, d, d, d]
        lib.vb_pathbuf_circle.argtypes = [vp, d, d, d, d]
        lib.vb_pathbuf_rounded_rect.argtypes = [vp, d, d, d, d, d, d]
        lib.vb_pathbuf_ellipse.argtypes = [vp, d, d, d, d, d, d]
        lib.vb_pathbuf_arc.argtypes = [vp, d, d, d, d, d, d, d, d]
        lib.vb_pathbuf_svg.argtypes = [vp, C.c_char_p]
        lib.vb_pathbuf_view.restype = _Path
        lib.vb_pathbuf_view.argtypes = [vp]
        _bound = True
    return lib


def _affine(t: Affine):
    return (C.c_double * 6)(*[float(v) for v in t.coeffs])


_VERB = {"M": ord("M"), "L": ord("L"), "Q": ord("Q"), "C": ord("C"), "Z": ord("Z")}


class NativeScene:
    def __init__(self):
        self.lib = _lib()
        self.handle = C.c_void_p(self.lib.vb_scene_new())
        self._keep = []  # buffers the C side refers to until resolve (image pixels)
        self._images = {}
        self._pixels = {}

    def __del__(self):
        if getattr(self, "handle", None):
            self.lib.vb_scene_free(self.handle)
            self.handle = None

    # -- marshalling ---------------------------------------------------------------------------------
    def _path(self, shape, tolerance: float):
        els = list(_shapes.path_elements(shape, tolerance))
        verbs = np.array([_VERB[e[0]] for e in els], dtype=np.uint8)
        coords = np.array([v for e in els for v in e[1:]], dtype=np.float64)
        p = _Path(verbs.ctypes.data, len(verbs), coords.ctypes.data)
        return p, (verbs, coords)

    @staticmethod
    def _color(c: Color) -> _Color:
        return _Color(c.r, c.g, c.b, c.a)

    def _image(self, im: Image) -> _Image:
        k = (id(im), im.key)
        if k not in self._images:  # the entry holds `im` too, so that its id cannot be reused by another Image meanwhile
            if im.key is not None:  # the key is the image's `pixels` (a host image's key points into its own data)
                self._pixels[("key", im.key)] = im.data
                ptr = im.key
            else:
                dk = id(im.data)  # one pixel buffer per blob: the atlas is keyed by it (image_cache.rs:113-114)
                if dk not in self._pixels:
                    self._pixels[dk] = np.ascontiguousarray(im.data, dtype=np.uint8).copy()
                ptr = self._pixels[dk].ctypes.data
            self._images[k] = (_Image(ptr, im.width, im.height, im.format, im.alpha_type, im.quality, im.x_extend, im.y_extend, im.alpha), im)
        return self._images[k][0]

    def _brush(self, brush):
        b = _Brush()
        hold = []
        if isinstance(brush, Color):
            b.kind = 0
            b.color = self._color(brush)
        elif isinstance(brush, Gradient):
            b.kind = {"linear": 1, "radial": 2, "sweep": 3}[brush.kind]
            for i, v in enumerate(brush.params):
                b.geom[i] = float(v)
            stops = (_Stop * max(len(brush.stops), 1))()
            for i, (o, c) in enumerate(brush.stops):
                stops[i] = _Stop(o, self._color(c))
            hold.append(stops)
            b.stops = C.cast(stops, C.c_void_p)
            b.n_stops = len(brush.stops)
            b.extend = brush.extend
            b.premul_interp = 1 if brush.premul_interp else 0
        elif isinstance(brush, Image):
            b.kind = 4
            img = self._image(brush)
            hold.append(img)
            b.image = C.cast(C.pointer(img), C.c_void_p)
        else:
            raise TypeError(type(brush))
        return b, hold

    @staticmethod
    def _stroke(s: Stroke) -> _Stroke:
        st = _Stroke(float(s.width), s.join, s.start_cap, s.end_cap, float(s.miter_limit), None, 0, float(s.dash_offset))
        if s.dash_pattern:
            arr = (C.c_double * len(s.dash_pattern))(*[float(d) for d in s.dash_pattern])
            st._keep = arr  # keeps the pattern alive as long as the struct
            st.dash_pattern = C.cast(arr, C.c_void_p)
            st.n_dashes = len(s.dash_pattern)
        return st

    def _check(self, rc):
        if rc != 0:
            raise ValueError(f"vb_scene call failed: {rc}")

    @property
    def n_draw_objects(self) -> int:
        """`vb_scene_n_draw_objects`: the draw objects encoded so far, as `Scene.n_draw_objects`."""
        return int(self.lib.vb_scene_n_draw_objects(self.handle))

    @property
    def n_points(self) -> int:
        """`vb_scene_n_points`: the path points encoded so far, as `Scene.n_points`."""
        return int(self.lib.vb_scene_n_points(self.handle))

    @property
    def n_stops(self) -> int:
        """`vb_scene_n_stops`: the gradient stops encoded so far, as `Scene.n_stops`."""
        return int(self.lib.vb_scene_n_stops(self.handle))

    @property
    def n_transforms(self) -> int:
        """`vb_scene_n_transforms`: the transform-stream entries encoded so far, as `Scene.n_transforms`."""
        return int(self.lib.vb_scene_n_transforms(self.handle))

    # -- vello::Scene surface ------------------------------------------------------------------------
    def fill(self, style: int, transform: Affine, brush, brush_transform: Optional[Affine], shape):
        p, hold = self._path(shape, 0.1)
        b, hb = self._brush(brush)
        bt = _affine(brush_transform) if brush_transform is not None else None
        self._check(self.lib.vb_scene_fill(self.handle, style, _affine(transform), C.byref(b), bt, C.byref(p)))

    def stroke(self, stroke: Stroke, transform: Affine, brush, brush_transform: Optional[Affine], shape):
        p, hold = self._path(shape, 0.01 if stroke.dash_pattern else 0.1)  # scene.rs:404-437: 0.01 only for the dash expansion
        b, hb = self._brush(brush)
        st = self._stroke(stroke)
        bt = _affine(brush_transform) if brush_transform is not None else None
        self._check(self.lib.vb_scene_stroke(self.handle, C.byref(st), _affine(transform), C.byref(b), bt, C.byref(p)))

    def _clip_args(self, clip_style, clip):
        if isinstance(clip_style, Stroke):
            st = self._stroke(clip_style)
            p, hold = self._path(clip, 0.01 if clip_style.dash_pattern else 0.1)
            return 0, C.byref(st), p, (st, hold)
        p, hold = self._path(clip, 0.1)
        return int(clip_style), None, p, hold

    def push_layer(self, clip_style, mix: int, compose: int, alpha: float, transform: Affine, clip):
        rule, st, p, hold = self._clip_args(clip_style, clip)
        self._check(self.lib.vb_scene_push_layer(self.handle, rule, st, mix, compose, alpha, _affine(transform), C.byref(p)))

    def push_luminance_mask_layer(self, clip_style, alpha: float, transform: Affine, clip):
        rule, st, p, hold = self._clip_args(clip_style, clip)
        self._check(self.lib.vb_scene_push_luminance_mask_layer(self.handle, rule, st, alpha, _affine(transform), C.byref(p)))

    def push_clip_layer(self, clip_style, transform: Affine, clip):
        rule, st, p, hold = self._clip_args(clip_style, clip)
        self._check(self.lib.vb_scene_push_clip_layer(self.handle, rule, st, _affine(transform), C.byref(p)))

    def pop_layer(self):
        self._check(self.lib.vb_scene_pop_layer(self.handle))

    def draw_image(self, image: Image, transform: Affine):
        img = self._image(image)
        self._check(self.lib.vb_scene_draw_image(self.handle, C.byref(img), _affine(transform)))

    def draw_blurred_rounded_rect(self, transform: Affine, rect, color: Color, radius: float, std_dev: float):
        r = (C.c_double * 4)(rect.x0, rect.y0, rect.x1, rect.y1)
        self._check(self.lib.vb_scene_draw_blurred_rounded_rect(self.handle, _affine(transform), r, self._color(color), float(radius), float(std_dev)))

    def draw_blurred_rounded_rect_in(self, shape, transform: Affine, rect, color: Color, radius: float, std_dev: float):
        p, hold = self._path(shape, 0.1)
        r = (C.c_double * 4)(rect.x0, rect.y0, rect.x1, rect.y1)
        self._check(self.lib.vb_scene_draw_blurred_rounded_rect_in(self.handle, C.byref(p), _affine(transform), r, self._color(color),
                                                                    float(radius), float(std_dev)))

    def append(self, other: "NativeScene", transform: Optional[Affine] = None):
        self._keep.append(other)  # its image buffers must outlive this scene's resolve
        self._check(self.lib.vb_scene_append(self.handle, other.handle, _affine(transform) if transform is not None else None))

    def batch(self, scenes) -> list:
        """`vb_scene_batch`: make this scene the batch of `scenes` (for `Renderer.set_cells`) and return its draw-object
        offsets (len(scenes) + 1 entries)."""
        scenes = list(scenes)
        self._keep = list(scenes)  # their image buffers must outlive this scene's resolve
        self._images, self._pixels = {}, {}
        arr = (C.c_void_p * max(len(scenes), 1))(*[s.handle for s in scenes])
        offs = (C.c_uint32 * (len(scenes) + 1))()
        self._check(self.lib.vb_scene_batch(self.handle, arr, len(scenes), offs))
        return [int(v) for v in offs]

    # -- Resolver::resolve ---------------------------------------------------------------------------
    def upload_device(self, renderer) -> Layout:
        """Resolve this scene ON THE DEVICE of `renderer` (vb_scene_upload_streams: the six streams are copied to their Layout
        offsets, kernels apply the patches / padding and generate the gradient ramps) and leave it uploaded there."""
        L = _Layout()
        self._check(self.lib.vb_scene_upload_device(renderer.handle, self.handle, C.byref(L)))
        renderer._cells = 1  # a new scene is one cell (Renderer.hit_map's whole frame)
        return Layout(L.n_draw_objects, L.n_paths, L.n_clips, L.bin_data_start, L.path_tag_base, L.path_data_base, L.draw_tag_base,
                      L.draw_data_base, L.transform_base, L.style_base)

    def resolve(self) -> Packed:
        pk = _Packed()
        self._check(self.lib.vb_scene_resolve(self.handle, C.byref(pk)))
        n_words = pk.scene_len // 4
        scene = np.ctypeslib.as_array(C.cast(pk.scene, C.POINTER(C.c_uint32)), shape=(n_words,)).copy() if n_words else np.zeros(0, np.uint32)
        if pk.ramp_h:
            ramps = np.ctypeslib.as_array(C.cast(pk.ramps, C.POINTER(C.c_uint32)), shape=(pk.ramp_h, pk.ramp_w)).copy()
        else:
            ramps = np.zeros((0, 512), dtype=np.uint32)
        atlas = np.ctypeslib.as_array(C.cast(pk.atlas, C.POINTER(C.c_uint8)), shape=(pk.atlas_h, pk.atlas_w, 4)).copy()
        L = pk.layout
        layout = Layout(L.n_draw_objects, L.n_paths, L.n_clips, L.bin_data_start, L.path_tag_base, L.path_data_base, L.draw_tag_base,
                        L.draw_data_base, L.transform_base, L.style_base)
        return Packed(scene=scene, layout=layout, ramps=ramps, atlas=atlas)


class NativePath:
    """vb_pathbuf: a growable kurbo-style path with the shape -> Bezier conversions done natively."""

    def __init__(self):
        self.lib = _lib()
        self.handle = C.c_void_p(self.lib.vb_pathbuf_new())

    def __del__(self):
        if getattr(self, "handle", None):
            self.lib.vb_pathbuf_free(self.handle)
            self.handle = None

    def add(self, shape, tolerance: float = 0.1) -> "NativePath":
        L = self.lib
        if isinstance(shape, _shapes.Rect):
            L.vb_pathbuf_rect(self.handle, shape.x0, shape.y0, shape.x1, shape.y1)
        elif isinstance(shape, _shapes.Line):
            L.vb_pathbuf_line(self.handle, shape.x0, shape.y0, shape.x1, shape.y1)
        elif isinstance(shape, _shapes.Circle):
            L.vb_pathbuf_circle(self.handle, shape.cx, shape.cy, shape.r, tolerance)
        elif isinstance(shape, _shapes.RoundedRect):
            L.vb_pathbuf_rounded_rect(self.handle, shape.x0, shape.y0, shape.x1, shape.y1, shape.radius, tolerance)
        elif isinstance(shape, _shapes.Ellipse):
            L.vb_pathbuf_ellipse(self.handle, shape.cx, shape.cy, shape.rx, shape.ry, shape.x_rotation, tolerance)
        elif isinstance(shape, _shapes.Arc):
            L.vb_pathbuf_arc(self.handle, shape.cx, shape.cy, shape.rx, shape.ry, shape.start_angle, shape.sweep_angle, shape.x_rotation, tolerance)
        else:
            for e in _shapes.path_elements(shape, tolerance):
                {"M": L.vb_pathbuf_move_to, "L": L.vb_pathbuf_line_to, "Q": L.vb_pathbuf_quad_to, "C": L.vb_pathbuf_curve_to}.get(
                    e[0], lambda h: L.vb_pathbuf_close(h))(self.handle, *[float(v) for v in e[1:]])
        return self

    def svg(self, d: str) -> "NativePath":
        if self.lib.vb_pathbuf_svg(self.handle, d.encode()) != 0:
            raise ValueError("bad SVG path data")
        return self

    def elements(self):
        """The path as ("M", x, y) ... tuples, like vello_b200.shapes.path_elements."""
        v = self.lib.vb_pathbuf_view(self.handle)
        verbs = bytes((C.c_uint8 * v.n_verbs).from_address(v.verbs)) if v.n_verbs else b""
        n = sum({77: 2, 76: 2, 81: 4, 67: 6, 90: 0}[b] for b in verbs)
        coords = list((C.c_double * n).from_address(v.coords)) if n else []
        out, i = [], 0
        for b in verbs:
            k = {77: 2, 76: 2, 81: 4, 67: 6, 90: 0}[b]
            out.append((chr(b),) + tuple(coords[i:i + k]))
            i += k
        return out
