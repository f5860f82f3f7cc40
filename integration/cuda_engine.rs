// cuda_engine.rs -- the reference-side binding of libvello_b200.so (drop next to vello/src/wgpu_engine.rs).
//
// UNCOMPILED SOURCE: this image has no Rust toolchain (`cargo --version` fails; wgpu / kurbo / peniko are not vendored), so the
// file documents, in the reference's own language, exactly what a vello maintainer adds. Every `extern "C"` item below is
// declared in include/vello_b200.h; the struct layouts are checked against that header by tests/test_abi.py on the C side.
//
// What it replaces:  Render::render_encoding_coarse + record_fine   vello/src/render.rs:135-629
//                    WgpuEngine::run_recording                      vello/src/wgpu_engine.rs:380-780
// What it keeps:     Scene, Renderer, RenderParams, AaConfig, Resolver (or its device twin, see `render_streams`).
#![allow(non_camel_case_types, dead_code)]
use std::os::raw::{c_char, c_int, c_void};

use vello_encoding::{Encoding, Layout, Resolver};

#[repr(C)]
pub struct VbOptions { pub device: i32, pub timing: u32, pub max_retries: u32, pub reserved: u32 }

/// == RenderParams (vello/src/lib.rs:357-369) + the stripe window extension
#[repr(C)]
#[derive(Default, Clone, Copy)]
pub struct VbParams {
    pub base_color: u32, pub width: u32, pub height: u32, pub aa: u32,
    pub bin_row0: u32, pub bin_row1: u32, pub tile_row0: u32, pub tile_row1: u32,
}

#[repr(C)]
#[derive(Default)]
pub struct VbFrameStats {
    pub failed: u32, pub binning: u32, pub ptcl: u32, pub tile: u32, pub seg_counts: u32, pub segments: u32, pub blend: u32, pub lines: u32,
    pub retries: u32, pub kernel_launches: u32, pub stage_ms: [f32; 11], pub total_ms: f32, pub arena_bytes: u64,
}

#[repr(C)] pub struct VbRampStop { pub offset: f32, pub r: f32, pub g: f32, pub b: f32, pub a: f32 }
#[repr(C)] pub struct VbRampPatch { pub draw_data_offset: u32, pub extend: u32, pub premul_interp: u32, pub n_stops: u32, pub stops: *const VbRampStop }
#[repr(C)] pub struct VbImagePatch { pub draw_data_offset: u32, pub width: u32, pub height: u32, pub pixels: *const u8 }
// one appended fragment of vb_compose: Encoding::append(&fragment, has_transform != 0 ? Some(transform) : None)
#[repr(C)] pub struct VbInstance { pub fragment: u32, pub has_transform: u32, pub transform: [f64; 6] }
/// == the six streams of vello_encoding::Encoding (encoding.rs:22-48) + its patches (resolve.rs:560-590)
#[repr(C)]
pub struct VbEncodingStreams {
    pub path_tags: *const u8, pub n_path_tags: u32,
    pub path_data: *const u32, pub n_path_data: u32,
    pub draw_tags: *const u32, pub n_draw_tags: u32,
    pub draw_data: *const u32, pub n_draw_data: u32,
    pub transforms: *const f32, pub n_transforms: u32,
    pub styles: *const u32, pub n_styles: u32,
    pub n_paths: u32, pub n_clips: u32, pub n_open_clips: u32,
    pub ramp_patches: *const VbRampPatch, pub n_ramp_patches: u32,
    pub image_patches: *const VbImagePatch, pub n_image_patches: u32,
}

/// a registered destination (vb_register_destination): VB_DEST_LINEAR 0 / VB_DEST_ARRAY 1, VB_DEST_RGBA8 0 / VB_DEST_BGRA8 1 /
/// VB_DEST_RGBA16F 2 / VB_DEST_RGBA32F 3, optionally | VB_DEST_PREMULTIPLIED 0x100 (premultiplied instead of straight alpha).
/// For a wgpu/Vulkan storage texture: the image's memory imported into CUDA, level 0 of its mipmapped array in `array`
/// (an Rgba16Float / R16G16B16A16_SFLOAT image takes VB_DEST_RGBA16F).
#[repr(C)]
pub struct VbDestination { pub kind: u32, pub format: u32, pub ptr: *mut c_void, pub row_pitch_bytes: usize, pub array: *mut c_void, pub x: u32, pub y: u32 }

pub enum VbRenderer {}
pub enum VbGroup {}

#[link(name = "vello_b200")]
extern "C" {
    pub fn vb_renderer_new(opt: *const VbOptions, out: *mut *mut VbRenderer) -> c_int;
    pub fn vb_renderer_free(r: *mut VbRenderer);
    pub fn vb_strerror(code: c_int) -> *const c_char;
    pub fn vb_last_error(r: *mut VbRenderer) -> *const c_char;
    // vello_encoding::Layout is #[repr(C)] 10 x u32 (resolve.rs:16-39) == vb_layout: passed by pointer.
    pub fn vb_render(r: *mut VbRenderer, scene: *const u8, scene_len: usize, layout: *const Layout,
                     ramps: *const u32, ramp_w: u32, ramp_h: u32, atlas: *const u8, atlas_w: u32, atlas_h: u32,
                     params: *const VbParams, out: *mut c_void, out_is_device: u32, stats: *mut VbFrameStats) -> c_int;
    // three frames in flight for exporters that read every frame back (examples/headless/src/main.rs:188-210)
    pub fn vb_render_begin(r: *mut VbRenderer, scene: *const u8, scene_len: usize, layout: *const Layout,
                           ramps: *const u32, ramp_w: u32, ramp_h: u32, atlas: *const u8, atlas_w: u32, atlas_h: u32,
                           params: *const VbParams, out_host: *mut c_void, stats: *mut VbFrameStats) -> c_int;
    pub fn vb_readback_wait(r: *mut VbRenderer) -> c_int;
    // Resolver::resolve on the device: hand over the raw streams instead of a packed buffer
    pub fn vb_scene_upload_streams(r: *mut VbRenderer, e: *const VbEncodingStreams, layout_out: *mut Layout) -> c_int;
    pub fn vb_render_uploaded(r: *mut VbRenderer, params: *const VbParams, out: *mut c_void, out_is_device: u32, stats: *mut VbFrameStats) -> c_int;
    pub fn vb_set_occlusion_cull(r: *mut VbRenderer, on: c_int) -> c_int;
    // pan / zoom a resident scene: with_winit's per-frame `scene.append(&fragment, Some(transform))` becomes one upload of
    // the fragment and vb_set_view(transform.as_coeffs()) per frame (NULL clears the view)
    pub fn vb_set_view(r: *mut VbRenderer, affine: *const [f64; 6]) -> c_int;
    pub fn vb_group_set_view(g: *mut VbGroup, affine: *const [f64; 6]) -> c_int;
    pub fn vb_debug_graph_captures(r: *mut VbRenderer, captures: *mut u64) -> c_int;
    // compose frames on the device from resident fragments: a toolkit's per-frame `Scene::new()` + `scene.append(&fragment,
    // Some(transform))` per widget becomes one vb_fragment_upload per fragment and one vb_compose of (id, transform) pairs
    pub fn vb_fragment_upload(r: *mut VbRenderer, e: *const VbEncodingStreams, fragment_out: *mut u32) -> c_int;
    pub fn vb_fragment_free(r: *mut VbRenderer, fragment: u32) -> c_int;
    pub fn vb_compose(r: *mut VbRenderer, instances: *const VbInstance, n: u32, layout_out: *mut Layout, draw_offsets: *mut u32) -> c_int;
    // every frame reads instance k's transform from row k of device memory ([a b c d e f] f32, row_pitch_bytes apart), so a
    // simulation that writes its transforms on vb_stream moves the instances without a compose per frame; NULL unbinds
    pub fn vb_bind_instance_transforms(r: *mut VbRenderer, device_transforms: *const f32, n: u32, row_pitch_bytes: usize) -> c_int;
    // damage tracking: a frame into the same destination as the last one repaints only the damaged tiles (moved bound instances,
    // plus the x0 y0 x1 y1 pixel rectangles added for the next frame); vb_last_damage gives one byte per tile of the last frame
    pub fn vb_set_damage_tracking(r: *mut VbRenderer, on: c_int) -> c_int;
    pub fn vb_add_damage(r: *mut VbRenderer, rects: *const u32, n: u32) -> c_int;
    pub fn vb_last_damage(r: *mut VbRenderer, tile_mask: *mut u8, cap: usize, n_damaged: *mut u32) -> c_int;
    // frames straight into a storage texture (a CUDA array) or a pitched buffer: the key goes where out_device goes
    pub fn vb_register_destination(r: *mut VbRenderer, d: *const VbDestination, key_out: *mut *mut c_void) -> c_int;
    pub fn vb_unregister_destination(r: *mut VbRenderer, key: *mut c_void) -> c_int;
    // vb_compose, after which the next tracked frame repaints only the instances added, removed or changed since the composition
    // the last frame rendered (matched in order by fragment and transform); vb_compose itself makes the next frame full
    pub fn vb_recompose(r: *mut VbRenderer, instances: *const VbInstance, n: u32, layout_out: *mut Layout, draw_offsets: *mut u32) -> c_int;
    // with tracking on: each uploaded scene (vb_render, vb_scene_upload, vb_scene_upload_streams) is compared on the device with
    // the one the last frame rendered, and the next frame into a device destination repaints only the draw objects that changed
    pub fn vb_set_upload_diff(r: *mut VbRenderer, on: c_int) -> c_int;
    // one frame on several GPUs of one box
    pub fn vb_group_new(devices: *const i32, n: u32, opt: *const VbOptions, out: *mut *mut VbGroup) -> c_int;
    pub fn vb_group_free(g: *mut VbGroup);
    pub fn vb_group_render(g: *mut VbGroup, scene: *const u8, scene_len: usize, layout: *const Layout,
                           ramps: *const u32, ramp_w: u32, ramp_h: u32, atlas: *const u8, atlas_w: u32, atlas_h: u32,
                           params: *const VbParams, out: *mut c_void, out_is_device: u32, stats: *mut VbFrameStats) -> c_int;
}

#[derive(Debug)]
pub enum CudaError { Code(c_int) }

/// Sits where `WgpuEngine` sits: owned by `Renderer`, `Send` but not `Sync` (one host thread per renderer, lib.rs:351-352).
pub struct CudaEngine { raw: *mut VbRenderer, packed: Vec<u8> }
unsafe impl Send for CudaEngine {}

impl CudaEngine {
    /// `Renderer::new` (lib.rs:432-458). `RendererOptions::use_cpu` has no equivalent: there is no CPU fallback.
    pub fn new(device: i32) -> Result<Self, CudaError> {
        let opt = VbOptions { device, timing: 0, max_retries: 0, reserved: 0 };
        let mut raw = std::ptr::null_mut();
        let rc = unsafe { vb_renderer_new(&opt, &mut raw) };
        if rc != 0 { return Err(CudaError::Code(rc)); }
        Ok(Self { raw, packed: Vec::new() })
    }

    fn params(p: &crate::RenderParams) -> VbParams {
        VbParams {
            base_color: p.base_color.premultiply().to_rgba8().to_u32(), // config.rs:183
            width: p.width, height: p.height,
            aa: match p.antialiasing_method { crate::AaConfig::Area => 0, crate::AaConfig::Msaa8 => 1, crate::AaConfig::Msaa16 => 2 },
            ..Default::default()
        }
    }

    /// Body of `Renderer::render_to_texture` (lib.rs:474-515) with the host-side resolve kept as it is (render.rs:148).
    pub fn render(&mut self, resolver: &mut Resolver, encoding: &Encoding, params: &crate::RenderParams,
                  atlas_rgba8: &[u8], atlas_w: u32, atlas_h: u32, out_rgba8: &mut [u8]) -> Result<VbFrameStats, CudaError> {
        let (layout, ramps, _images) = resolver.resolve(encoding, &mut self.packed);
        let p = Self::params(params);
        let mut stats = VbFrameStats::default();
        let rc = unsafe {
            vb_render(self.raw, self.packed.as_ptr(), self.packed.len(), &layout, ramps.data.as_ptr(), ramps.width, ramps.height,
                      atlas_rgba8.as_ptr(), atlas_w, atlas_h, &p, out_rgba8.as_mut_ptr().cast(), 0, &mut stats)
        };
        // an arena overflow is grown-and-re-run inside the call; only a persisting one is an error (the reference leaves the
        // texture unwritten and says nothing, lib.rs:753-763)
        if rc != 0 { Err(CudaError::Code(rc)) } else { Ok(stats) }
    }

    /// Same frame without `Resolver::resolve` on the host: the streams go to the device as they are and are resolved there.
    pub fn render_streams(&mut self, e: &VbEncodingStreams, params: &crate::RenderParams, out_rgba8: &mut [u8]) -> Result<VbFrameStats, CudaError> {
        let mut layout = Layout::default();
        let rc = unsafe { vb_scene_upload_streams(self.raw, e, &mut layout) };
        if rc != 0 { return Err(CudaError::Code(rc)); }
        let p = Self::params(params);
        let mut stats = VbFrameStats::default();
        let rc = unsafe { vb_render_uploaded(self.raw, &p, out_rgba8.as_mut_ptr().cast(), 0, &mut stats) };
        if rc != 0 { Err(CudaError::Code(rc)) } else { Ok(stats) }
    }
}

impl Drop for CudaEngine {
    fn drop(&mut self) { unsafe { vb_renderer_free(self.raw) } }
}
