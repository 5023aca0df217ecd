// hk_kernels.h — host-callable launchers of the CUDA kernels (implemented in kernels_light.cu / kernels_post.cu / kernels_upscale.cu).
#pragma once
#include "hk_device.cuh"
#include "hk_tile.cuh"

// `wide`: the image-exact traversal mode (hk_wide.cuh) when the scene's 4-wide trees exist, else the reference's fixed-order walk
void hk_launch_gbuffer(const hkd::KParams& P, bool count, bool wide, cudaStream_t st);
void hk_launch_albedo(const hkd::KParams& P, cudaStream_t st);
void hk_launch_direct(const hkd::KParams& P, bool emissive, bool count, bool wide, cudaStream_t st);
void hk_launch_indirect(const hkd::KParams& P, bool multi, bool count, bool wide, cudaStream_t st);
// pooled (cooperative) form of the indirect pass: shared-memory ray pool, dynamic fetch, TMA-staged scene records (kernels_pool.cu)
void hk_launch_indirect_pool(const hkd::KParams& P, bool multi, bool count, cudaStream_t st);
void hk_launch_spatial(const hkd::KParams& P, bool emissive, const hkd::TileMap* depth_map, const hkd::TileMap* q3_map, const hkd::SpatialTable& table,
                       cudaStream_t st);
void hk_launch_extract_depth(const hkd::KParams& P, cudaStream_t st);   // depth plane <- pos_depth.w over the launch rectangle
void hk_launch_scatter_resolve(const hkd::KParams& P, int signal, cudaStream_t st);
void hk_launch_trace_rays(const hkd::DeviceScene& sc, const hk_ray* rays, size_t n, hk_hit* hits, bool wide, cudaStream_t st);

// post process: `signals` = 2 or 3 (post_process.rs:949-954)
void hk_launch_demodulation(const hkd::KParams& P, int signals, cudaStream_t st);
void hk_launch_denoise_level(const hkd::KParams& P, int level, int signals, bool fuse_tone_mapping, bool keep_denoised, const hkd::TileMap* maps, cudaStream_t st);
void hk_launch_tone_mapping(const hkd::KParams& P, cudaStream_t st);

// temporal upscalers (kernels_upscale.cu); full-frame contexts only
void hk_launch_smaa_tu4x(const hkd::KParams& P, cudaStream_t st);               // over col_lo..col_hi x row_lo..row_hi (render pixels)
void hk_launch_smaa_tu4x_extrapolate(const hkd::KParams& P, cudaStream_t st);
void hk_launch_taa_jasmine(const hkd::KParams& P, bool smaa, cudaStream_t st);  // over col_lo..col_hi x row_lo..row_hi = the output size
// FSR 1.0 (Upscale::Fsr1): over col_lo..col_hi x row_lo..row_hi = the camera target; full-frame contexts only
void hk_launch_fsr_easu(const hkd::KParams& P, cudaStream_t st);   // taa_output / tone-mapped (render size) -> upscale_output (W x H)
void hk_launch_fsr_rcas(const hkd::KParams& P, cudaStream_t st);   // upscale_output -> upscale_sharpen_output

// halo exchange between tiles of one frame (kernels_post.cu): copies the ten reservoir buffers of the global pixel rectangle
// [x0,x1) x [y0,y1) from `src`'s planes into `dst`'s planes; `src` may be peer memory
void hk_launch_halo_copy(const hkd::Planes& dst, const hkd::Band& dst_band, const hkd::Planes& src, const hkd::Band& src_band,
                         int x0, int x1, int y0, int y1, cudaStream_t st);
// the same for one Rgba16Float image stored over the tiles' allocations at `scale` x the render resolution
void hk_launch_halo_copy_image(uint2* dst, const hkd::Band& dst_band, const uint2* src, const hkd::Band& src_band, int scale,
                               int x0, int x1, int y0, int y1, cudaStream_t st);

// the per-frame half of the scene rebuilt on the device (kernels_scene.cu; hk_scene_update_transforms)
void hk_launch_scene_instances(uint32_t n, const float4* models, const float4* previous, const float* mesh_aabbs, hk_instance* instances,
                               hkd::hk_instance_trav* trav, float4* previous_out, uint32_t* moved_out, float4* box_lo, float4* box_hi, cudaStream_t st);
// bvh 0.7.1 BVH::build + flatten_custom over n boxes into out[0 .. 3n-2); every shape's tree-node index is written to
// index_base + shape * index_stride.  `scratch`: hk_scene_bvh_scratch_bytes(n) bytes.
void hk_launch_build_flat_bvh(uint32_t n, const float4* box_lo, const float4* box_hi, void* scratch, hk_node* out, void* index_base,
                              uint32_t index_stride, cudaStream_t st);
size_t hk_scene_bvh_scratch_bytes(uint32_t n);
// the 4-wide TLAS (hk_wide.cuh) of the flat TLAS flat[0 .. 3n-2) over n instances, as wide_build.h derives it: at most n - 1 nodes,
// n ranks, and state = {ready, stack need of the whole walk, node count} where ready = blas_ok && the tree could be derived
// && its need + base_need <= HK_WIDE_STACK.  `scratch`: hk_wide_tlas_scratch_bytes(n) bytes.
void hk_launch_build_wide_tlas(uint32_t n, const hk_node* flat, bool blas_ok, uint32_t base_need, void* scratch, hkd::hk_wide_node* nodes,
                               uint32_t* rank, uint32_t* state, cudaStream_t st);
size_t hk_wide_tlas_scratch_bytes(uint32_t n);
// GpuMesh::try_from (mod.rs:379-467) on the device for a batch of meshes (hk_scene_add_meshes): per mesh, where its staged
// attributes and indices start, which topology it has, and where its records go in the scene's buffers.  Shapes (primitives) are
// numbered across the batch; jobs are in batch order.
struct MeshJob {
    uint32_t src_vertex, src_index, indexed, strip;        // staged positions / normals / uvs from src_vertex, indices from src_index
    uint32_t shape_begin, shapes;                           // the mesh's primitives in the batch
    uint32_t dst_vertex, dst_primitive, dst_node;           // first record in the scene's vertex / primitive / BLAS buffers
};
// packs the vertices and primitives of the batch and builds every mesh's BLAS (bvh 0.7.1, as host/hikari.cpp build_flat_bvh with no
// node-index write-back) into nodes[dst_node ..); `scratch`: hk_blas_scratch_bytes(total_primitives).  Returns the launch count.
int hk_launch_build_meshes(uint32_t n_jobs, const MeshJob* jobs, uint32_t total_vertices, uint32_t total_primitives, const float* positions,
                           const float* normals, const float* uvs, const uint32_t* indices, void* scratch, hk_vertex* vertices,
                           hk_primitive* primitives, hk_node* nodes, cudaStream_t st);
size_t hk_blas_scratch_bytes(uint32_t primitives);
void hk_launch_scene_emissives(uint32_t ne, hk_emissive* emissives, const hk_instance* instances, const hk_material* materials,
                               const hk_primitive* primitives, const hk_vertex* vertices, float4* box_lo, float4* box_hi, cudaStream_t st);
