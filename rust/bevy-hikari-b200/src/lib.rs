//! Render-graph nodes that replace the bodies of bevy-hikari's `PrepassNode`, `LightNode` and `PostProcessNode`
//! (reference: src/prepass.rs:769-851, src/light.rs:590-702, src/post_process.rs:1140-1311) with calls into
//! libhikari_b200 through `hikari-b200-sys`.  Everything else of the plugin — `HikariSettings`, `Taa`, `Upscale`, `graph::NAME`,
//! the Extract / Prepare systems that fill the nine storage buffers — stays the reference's own Rust.
//!
//! STATUS: written against the generated declarations of `hikari-b200-sys` and Bevy 0.9's render-graph API, NOT COMPILED — the
//! repository's build container has no Rust toolchain (INTEGRATION.md).  The host logic this file would contain is exercised
//! through its C++ mirror (bevy_hikari_b200/host/), which binds the same C ABI.
use std::ffi::CStr;

use bevy::{
    prelude::*,
    render::{
        render_graph::{Node, NodeRunError, RenderGraphContext, SlotInfo, SlotType},
        renderer::RenderContext,
        view::ExtractedView,
    },
};
use bevy_hikari::{prelude::*, view::{FrameUniform, PreviousViewUniform}};
use hikari_b200_sys as ffi;

/// The scene buffers of the render world, ONE for every camera: the reference's `MeshMaterialBindGroup` is a single resource
/// (src/mesh_material/mod.rs:677-681) that every camera's `LightNode` binds (src/light.rs:641-642).  Uploaded and animated once per
/// frame; each camera's context attaches to it (include/hikari_b200.h: hk_shared_scene).  Dropping it drops the handle only: the
/// device memory goes with the last camera context that renders it.
#[derive(Resource)]
pub struct HikariB200Scene(pub *mut ffi::hk_shared_scene);
unsafe impl Send for HikariB200Scene {}
unsafe impl Sync for HikariB200Scene {}

impl FromWorld for HikariB200Scene {
    fn from_world(_world: &mut World) -> Self {
        let mut scene = std::ptr::null_mut();
        // a stream of its own: cameras on other streams are ordered against it by the library
        if unsafe { ffi::hk_shared_scene_create(&mut scene, 0, std::ptr::null_mut()) } != ffi::HK_OK {
            error!("hk_shared_scene_create: {}", scene_error(std::ptr::null_mut()));
        }
        HikariB200Scene(scene)
    }
}

impl Drop for HikariB200Scene {
    fn drop(&mut self) {
        unsafe { ffi::hk_shared_scene_destroy(self.0) }
    }
}

/// One `hk_context` per camera entity (what `ReservoirCache` + the texture caches are in the reference, src/light.rs:307-383).
#[derive(Component)]
pub struct HikariB200Context(pub *mut ffi::hk_context);
unsafe impl Send for HikariB200Context {}
unsafe impl Sync for HikariB200Context {}

impl Drop for HikariB200Context {
    fn drop(&mut self) {
        unsafe { ffi::hk_context_destroy(self.0) }
    }
}

/// `prepare_light_textures` / `prepass_textures_system` / `prepare_post_process_textures` collapse into create-or-resize; a new
/// camera's context is attached to the render world's one scene (only reservoirs and textures are per camera, src/light.rs:69).
pub fn prepare_contexts(
    mut commands: Commands,
    scene: Res<HikariB200Scene>,
    cameras: Query<(Entity, &ExtractedCamera, Option<&HikariB200Context>), With<HikariSettings>>,
) {
    for (entity, camera, context) in &cameras {
        let Some(size) = camera.physical_target_size else { continue };
        match context {
            Some(context) => unsafe {
                // zeroes the temporal state when the size changed, like the re-allocation in src/light.rs:342-363
                ffi::hk_context_resize(context.0, size.x, size.y, 0, size.y);
            },
            None => {
                let mut ctx = std::ptr::null_mut();
                let rc = unsafe { ffi::hk_context_create(&mut ctx, 0, size.x, size.y, 0, size.y, std::ptr::null_mut()) };
                if rc != ffi::HK_OK {
                    error!("hk_context_create: {}", last_error(std::ptr::null_mut()));
                    continue;
                }
                if unsafe { ffi::hk_context_attach_scene(ctx, scene.0) } != ffi::HK_OK {
                    error!("hk_context_attach_scene: {}", last_error(ctx));
                }
                commands.entity(entity).insert(HikariB200Context(ctx));
            }
        }
    }
}

fn scene_error(scene: *mut ffi::hk_shared_scene) -> String {
    unsafe { CStr::from_ptr(ffi::hk_shared_scene_last_error(scene)) }.to_string_lossy().into_owned()
}

fn last_error(ctx: *mut ffi::hk_context) -> String {
    unsafe { CStr::from_ptr(ffi::hk_last_error(ctx)) }.to_string_lossy().into_owned()
}

/// What bind group 0 carries each frame (src/prepass.rs:81-125, src/light.rs:630-639) + the settings that select passes.
pub fn frame_inputs(
    frame: &FrameUniform,
    view: &ExtractedView,
    previous_view: &PreviousViewUniform,
    lights: &bevy::pbr::GpuLights,
    settings: &HikariSettings,
) -> ffi::hk_frame_inputs {
    // FrameUniform (src/view.rs:105-123) already is the 256-byte std140 image hk_frame_uniform declares
    let frame: ffi::hk_frame_uniform = unsafe { std::mem::transmute_copy(frame) };
    let view_proj = view.projection * view.transform.compute_matrix().inverse();
    ffi::hk_frame_inputs {
        frame,
        view: ffi::hk_view {
            view_proj: view_proj.to_cols_array(),
            inverse_view_proj: view_proj.inverse().to_cols_array(),
            view: view.transform.compute_matrix().to_cols_array(),
            inverse_view: view.transform.compute_matrix().inverse().to_cols_array(),
            projection: view.projection.to_cols_array(),
            inverse_projection: view.projection.inverse().to_cols_array(),
            world_position: view.transform.translation().to_array(),
            _pad0: 0.0,
            viewport: view.viewport.as_vec4().to_array(),
        },
        previous_view: unsafe { std::mem::transmute_copy(previous_view) },   // { view_proj, inverse_view_proj }, src/view.rs:31-35
        lights: ffi::hk_lights {
            directional_color: lights.directional_lights[0].color.to_array(),
            direction_to_light: lights.directional_lights[0].dir_to_light.to_array(),
            _pad0: 0.0,
            ambient_color: lights.ambient_color.to_array(),
        },
        denoise: settings.denoise as u32,
        taa_jitter: matches!(settings.taa, Taa::Jasmine) as u32,                 // src/prepass.rs:193-196
        smaa_tu4x: matches!(settings.upscale, Upscale::SmaaTu4x { .. }) as u32,  // src/prepass.rs:197-199
        temporal_upscalers: 1,
        fsr1: matches!(settings.upscale, Upscale::Fsr1 { .. }) as u32,           // src/post_process.rs:1279
        fsr_sharpness: settings.upscale.sharpness(),
    }
}

macro_rules! hikari_node {
    ($name:ident, $call:path, $doc:literal) => {
        #[doc = $doc]
        pub struct $name {
            query: QueryState<(
                &'static FrameUniform,
                &'static ExtractedView,
                &'static PreviousViewUniform,
                &'static HikariSettings,
                &'static HikariB200Context,
            )>,
        }
        impl $name {
            pub const IN_VIEW: &'static str = "view";
            pub fn new(world: &mut World) -> Self {
                Self { query: world.query_filtered() }
            }
        }
        impl Node for $name {
            fn input(&self) -> Vec<SlotInfo> {
                vec![SlotInfo::new(Self::IN_VIEW, SlotType::Entity)]
            }
            fn update(&mut self, world: &mut World) {
                self.query.update_archetypes(world);
            }
            fn run(&self, graph: &mut RenderGraphContext, _render_context: &mut RenderContext, world: &World) -> Result<(), NodeRunError> {
                let entity = graph.get_input_entity(Self::IN_VIEW)?;
                // missing inputs: return Ok(()) and skip, like the reference nodes (src/light.rs:606-617)
                let Ok((frame, view, previous_view, settings, context)) = self.query.get_manual(world, entity) else { return Ok(()) };
                let Some(lights) = world.get_resource::<bevy::pbr::GpuLights>() else { return Ok(()) };
                let inputs = frame_inputs(frame, view, previous_view, lights, settings);
                match unsafe { $call(context.0, &inputs) } {
                    ffi::HK_OK | ffi::HK_ERR_NOT_READY => {}
                    _ => error!("{}: {}", stringify!($call), last_error(context.0)),
                }
                Ok(())
            }
        }
    };
}

hikari_node!(PrepassNode, ffi::hk_prepass_run, "Replaces `PrepassNode::run` (src/prepass.rs:769-851): primary rays instead of the raster pass.");
hikari_node!(LightNode, ffi::hk_light_run, "Replaces `LightNode::run` (src/light.rs:590-702): albedo, both direct passes, indirect, spatial reuse.");
hikari_node!(PostProcessNode, ffi::hk_post_process_run, "Replaces `PostProcessNode::run` (src/post_process.rs:1140-1311): denoise, tone mapping, SMAA TU4x / TAA / FSR1.");

/// Hands the nine storage buffers of bind group 2 (src/mesh_material/mod.rs:684-808) to the device whenever any of them changed —
/// once per frame for every camera, into the shared scene.
/// The encase byte images are `#[repr(C)]`-compatible with include/hk_layout.h (static_asserts there, size assertions in the -sys crate).
pub fn upload_scene(scene: &HikariB200Scene, desc: &ffi::hk_scene_desc, instances_only: bool) {
    let rc = unsafe {
        if instances_only { ffi::hk_shared_scene_update_instances(scene.0, desc) } else { ffi::hk_shared_scene_upload(scene.0, desc) }
    };
    if rc != ffi::HK_OK {
        error!("scene upload: {}", scene_error(scene.0));
    }
}

/// Frames on which only `GlobalTransform`s changed (the common case of an animated scene): the per-frame half of the scene —
/// instance AABBs and matrices, TLAS, emissives, emissive BVH — is rebuilt ON THE DEVICE from one matrix per instance, once for
/// every camera (include/hikari_b200.h: hk_shared_scene_update_transforms; replaces the CPU work of src/mesh_material/instance.rs:352-437).
/// `models` / `previous_models`: `GlobalTransform::compute_matrix().to_cols_array()` of every instance in instance order and its
/// `GlobalTransformQueue[1]`; `mesh_aabbs`: `[center.x, center.y, center.z, half.x, half.y, half.z]` of each instance's mesh `Aabb`.
/// The caller keeps the reference's conditions for the full path (instance set changed, or an emissive's scale left its cached alias
/// table's +-0.01 range, instance.rs:385-397) and calls `upload_scene(.., instances_only = true)` then.  A model with an infinite
/// or NaN entry is refused here and by `upload_scene` (`HK_ERR_INVALID_ARGUMENT`, logged with the instance it names): the scene
/// stays as it was.
pub fn update_transforms(scene: &HikariB200Scene, models: &[[f32; 16]], previous_models: Option<&[[f32; 16]]>, mesh_aabbs: &[[f32; 6]]) -> bool {
    debug_assert!(models.len() == mesh_aabbs.len() && previous_models.map_or(true, |p| p.len() == models.len()));
    let rc = unsafe {
        ffi::hk_shared_scene_update_transforms(scene.0, models.as_ptr() as *const f32, previous_models.map_or(std::ptr::null(), |p| p.as_ptr() as *const f32),
                                               mesh_aabbs.as_ptr() as *const f32, models.len() as u32)
    };
    match rc {
        ffi::HK_OK => true,
        ffi::HK_ERR_UNSUPPORTED => false,      // a TLAS that is not in bvh 0.7.1's layout: keep the host path
        _ => { error!("hk_shared_scene_update_transforms: {}", scene_error(scene.0)); false }
    }
}

/// The image the overlay pass presents (src/overlay.rs:226-231): a CUDA device pointer, to be imported into the swap-chain API
/// through external memory (with `cudarc`: `CudaSlice::from_raw`).
pub fn presented_image(ctx: &HikariB200Context, settings: &HikariSettings) -> Option<(*mut std::ffi::c_void, usize)> {
    let which = match (settings.upscale, settings.taa) {
        (Upscale::Fsr1 { .. }, _) => ffi::HK_OUT_FSR_SHARPENED,
        (Upscale::SmaaTu4x { .. }, Taa::None) => ffi::HK_OUT_UPSCALED,
        (Upscale::SmaaTu4x { .. }, Taa::Jasmine) => ffi::HK_OUT_TAA,
    };
    let (mut ptr, mut bytes) = (std::ptr::null_mut(), 0usize);
    (unsafe { ffi::hk_get_output(ctx.0, which, &mut ptr, &mut bytes) } == ffi::HK_OK).then_some((ptr, bytes))
}
