/*
 * nvblox_b200.h -- C-ABI of the H100-native depth-integration hot path.
 *
 * This is the drop-in boundary for ONE path of nvblox_core:
 *   ViewCalculator::getBlocksInImageViewRaycast  ->
 *   ProjectiveTsdfIntegrator::integrateFrame     ->
 *   EsdfIntegrator::integrateBlocks
 * as driven by nvblox::Mapper::integrateDepth / Mapper::updateEsdf.
 *
 * The reference exposes this path as a C++ ABI (libnvblox_lib.so + Eigen-typed
 * headers). The library below is the C core a source-compatible `nvblox/...`
 * header set forwards to (see INTEGRATION.md and include/nvblox/): plain
 * pointers and sizes only, no Eigen / torch / STL types in any signature.
 *
 * Citations: paths are relative to
 *   nvblox_ros/nvblox_core/nvblox/ of isaac_ros_nvblox   ("C/" in SURVEY.md)
 *
 * Conventions
 *   - Every function returns NVB_OK (0) or a negative NvbStatus; the message of
 *     the last failure on the calling thread is nvb_last_error(). (The reference
 *     aborts the process through glog CHECK on the same conditions,
 *     C/include/nvblox/core/internal/error_check.h:28-65; the C++ mirror in
 *     include/nvblox/ turns a non-zero status back into an abort.)
 *   - Transforms are 16 floats, 4x4 column-major = Eigen::Isometry3f::data()
 *     (C/include/nvblox/core/types.h:141-153).
 *   - Block indices are int32 triples (Index3D = Eigen::Vector3i).
 *   - Voxel layouts in device memory are the reference's
 *     (C/include/nvblox/map/voxels.h:28-74, blox.h:28-67): a block is
 *     voxels[8][8][8], z fastest; TsdfVoxel 8 B. The ESDF layer is the
 *     exception: a device block of 10 240 B holds its 512 voxels (z fastest)
 *     as 512 16-byte cells {squared_distance_vox, parent_direction[3]} and
 *     then 512 flag words (bytes is_inside, observed, is_site, pad). Every
 *     host-facing copy (get/set blocks, map files, voxel queries) is in
 *     20-byte NvbEsdfVoxel records.
 *   - Functions without the _async suffix are synchronous at return, like the
 *     reference (projective_integrator_impl.cuh:305, esdf_integrator.cu:258).
 *   - One NvbMapper is driven from one host thread (same as nvblox::Mapper).
 */
#ifndef NVBLOX_B200_H_
#define NVBLOX_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(_WIN32)
#define NVB_API
#else
#define NVB_API __attribute__((visibility("default")))
#endif

typedef enum {
  NVB_OK = 0,
  NVB_ERR_INVALID_ARGUMENT = -1,
  NVB_ERR_CUDA = -2,
  NVB_ERR_CAPACITY = -3,      /* a slab / hash could not be grown */
  NVB_ERR_INDEX_RANGE = -4,   /* a block index does not fit the 21-bit hash key */
  NVB_ERR_NO_DEVICE = -5,
  NVB_ERR_IO = -6             /* a map file could not be opened, read or written, or libsqlite3.so.0 is missing */
} NvbStatus;

/* Where a caller buffer lives. */
typedef enum { NVB_MEM_HOST = 0, NVB_MEM_DEVICE = 1 } NvbMemory;

/* Layers of the map (C/include/nvblox/map/common_names.h TsdfLayer / EsdfLayer). */
typedef enum { NVB_LAYER_TSDF = 0, NVB_LAYER_ESDF = 1, NVB_LAYER_OCCUPANCY = 2, NVB_LAYER_FREESPACE = 3, NVB_LAYER_COLOR = 4, NVB_LAYER_MESH = 5 } NvbLayer;

/* ProjectiveLayerType of a Mapper (C/include/nvblox/mapper/mapper.h:40-48): which layer integrateDepth feeds. */
typedef enum {
  NVB_PROJECTIVE_TSDF = 0,
  NVB_PROJECTIVE_OCCUPANCY = 1,
  NVB_PROJECTIVE_TSDF_WITH_FREESPACE = 2 /* TSDF + FreespaceLayer (dynablox), used by the ESDF to ignore free voxels */
} NvbProjectiveLayerType;

/* nvblox::Camera (C/include/nvblox/sensors/camera.h:193-203) with its
 * std::optional<RadialTangentialDistortionParams> (C/include/nvblox/sensors/distortion.h:24-62):
 * has_distortion = 0 is std::nullopt. */
typedef struct {
  float fu, fv, cu, cv;
  int32_t width, height;
  int32_t has_distortion;
  float k1, k2, k3, k4, k5, k6; /* radial: numerator k1..k3, denominator k4..k6 */
  float p1, p2;                 /* tangential */
} NvbCamera;

/* WeightingFunctionType (C/include/nvblox/integrators/weighting_function.h:11-18). */
typedef enum {
  NVB_WEIGHT_CONSTANT = 0,
  NVB_WEIGHT_CONSTANT_DROPOFF = 1,
  NVB_WEIGHT_INVERSE_SQUARE = 2,
  NVB_WEIGHT_INVERSE_SQUARE_DROPOFF = 3,
  NVB_WEIGHT_INVERSE_SQUARE_TSDF_DISTANCE_PENALTY = 4,
  NVB_WEIGHT_LINEAR_WITH_MAX = 5
} NvbWeighting;

/* WorkspaceBoundsType (C/include/nvblox/geometry/workspace_bounds.h:24). */
typedef enum { NVB_WS_UNBOUNDED = 0, NVB_WS_HEIGHT_BOUNDS = 1, NVB_WS_BOUNDING_BOX = 2 } NvbWorkspaceBounds;

/* MaskMode (C/include/nvblox/sensors/image.h:383). */
typedef enum { NVB_MASK_NON_INVERTED = 0, NVB_MASK_INVERTED = 1 } NvbMaskMode;

/* ProjectiveIntegrator / ProjectiveTsdfIntegrator / ViewCalculator parameters
 * (C/include/nvblox/integrators/projective_integrator_params.h:24-63,
 *  view_calculator_params.h:22-60). */
typedef struct {
  float truncation_distance_vox;    /* 4   */
  float max_integration_distance_m; /* 7   */
  float max_weight;                 /* 5   */
  float invalid_depth_decay_factor; /* -1 (off) */
  int32_t weighting_type;           /* NVB_WEIGHT_INVERSE_SQUARE */
  int32_t raycast_subsampling;      /* 4   */
  int32_t workspace_bounds_type;    /* NVB_WS_UNBOUNDED */
  float workspace_min[3];
  float workspace_max[3];
} NvbTsdfParams;

/* EsdfIntegrator parameters (C/include/nvblox/integrators/esdf_integrator_params.h:22-31). */
typedef struct {
  float max_esdf_distance_m;   /* 2    */
  float max_site_distance_vox; /* 1    */
  float min_weight;            /* 1e-4 */
  float occupied_threshold;    /* 0.5: probability above which an occupancy voxel is inside an obstacle
                                  (EsdfIntegrator::occupied_threshold, esdf_integrator.h:198,219,375) */
} NvbEsdfParams;

/* ProjectiveOccupancyIntegrator's inverse sensor model
 * (C/include/nvblox/integrators/occupancy_integrator_params.h:21-40). */
typedef struct {
  float free_region_occupancy_probability;       /* 0.3 */
  float occupied_region_occupancy_probability;   /* 0.7 */
  float unobserved_region_occupancy_probability; /* 0.5 */
  float occupied_region_half_width_m;            /* 0.1 */
} NvbOccupancyParams;

/* TsdfVoxel as stored in HBM, EsdfVoxel as copied to and from the host (C/include/nvblox/map/voxels.h:28-34,55-74). */
typedef struct {
  float distance;
  float weight;
} NvbTsdfVoxel;

typedef struct {
  float squared_distance_vox;
  int32_t parent_direction[3];
  uint8_t is_inside, observed, is_site, pad_;
} NvbEsdfVoxel;

/* FreespaceVoxel (C/include/nvblox/map/voxels.h:38-52): two nvblox::Time (int64 milliseconds) and a bool. */
typedef struct {
  int64_t last_occupied_timestamp_ms;
  int64_t consecutive_occupancy_duration_ms;
  uint8_t is_high_confidence_freespace, pad_[7];
} NvbFreespaceVoxel;

/* ColorVoxel (C/include/nvblox/map/voxels.h:77-83): Color = 3 bytes RGB (core/color.h:28-68), one byte of padding, float weight.
 * A freshly allocated block holds ColorVoxel() = Color::Gray() (127, 127, 127), weight 0. */
typedef struct {
  uint8_t r, g, b, pad_;
  float weight;
} NvbColorVoxel;

/* Construction options. capacity = number of 8x8x8 blocks each layer's slab is
 * sized for up front (it grows by doubling, which is a synchronising event;
 * BlockMemoryPool does the same, C/include/nvblox/map/internal/impl/
 * block_memory_pool_impl.h:30-73). 0 selects the default (65536). */
typedef struct {
  float voxel_size_m;
  int32_t device;                /* CUDA device ordinal */
  int32_t tsdf_capacity_blocks;
  int32_t esdf_capacity_blocks;
  int32_t esdf_persistent;       /* how computeEsdf runs. 3 (default): exchange-slab wavefront, whole update in one cooperative
                                    launch, one grid barrier per ring (adds two ESDF-sized slabs + the candidate records);
                                    1: four-phase wavefront, one cooperative launch, four barriers per ring;
                                    2: gather-replay wavefront, two barriers per ring (DESIGN.md section 6);
                                    0: one launch per ring phase with a host-read counter, like the reference */
  int32_t projective_layer_type; /* NvbProjectiveLayerType: TSDF (default) or occupancy */
  int32_t keep_last_view;        /* 1: every integrated frame leaves a device copy of its depth image, pose and camera
                                    behind for nvb_mapper_decay_exclude_last_view, like Mapper::integrateDepth does
                                    (mapper_impl.h:70-78); 0 (default): no copy, pass the view to nvb_mapper_decay */
} NvbMapperOptions;

/* = nvblox::Mapper restricted to {TsdfLayer, EsdfLayer, ProjectiveTsdfIntegrator,
 * EsdfIntegrator, BlocksToUpdateTracker(kEsdf)} (C/include/nvblox/mapper/mapper.h:107-836). */
typedef struct NvbMapper NvbMapper;

NVB_API const char* nvb_last_error(void);
NVB_API const char* nvb_version(void);
/* Number of CUDA devices visible (0 if none / no driver). */
NVB_API int32_t nvb_device_count(void);

NVB_API void nvb_default_mapper_options(NvbMapperOptions* opts);
NVB_API void nvb_default_tsdf_params(NvbTsdfParams* p);
NVB_API void nvb_default_esdf_params(NvbEsdfParams* p);

/* Mapper::Mapper(voxel_size_m, ...) (mapper.h:119-124). */
NVB_API int32_t nvb_mapper_create(const NvbMapperOptions* opts, NvbMapper** out);
NVB_API void nvb_mapper_destroy(NvbMapper* m);
/* LayerCake::clear + tracker reset. */
NVB_API int32_t nvb_mapper_clear(NvbMapper* m);
/* Mapper::tsdf_integrator().<setters> (projective_tsdf_integrator.h:59-121,
 * projective_integrator.h:56-85, view_calculator.h:88-145). */
NVB_API int32_t nvb_mapper_set_tsdf_params(NvbMapper* m, const NvbTsdfParams* p);
NVB_API int32_t nvb_mapper_get_tsdf_params(const NvbMapper* m, NvbTsdfParams* p);
/* Mapper::esdf_integrator().<setters> (esdf_integrator.h:178-283). */
NVB_API int32_t nvb_mapper_set_esdf_params(NvbMapper* m, const NvbEsdfParams* p);
NVB_API int32_t nvb_mapper_get_esdf_params(const NvbMapper* m, NvbEsdfParams* p);
/* Mapper::occupancy_integrator().<setters> (C/include/nvblox/integrators/projective_occupancy_integrator.h:57-88).
 * With an occupancy mapper, nvb_mapper_integrate_depth runs ProjectiveOccupancyIntegrator::integrateFrame
 * (same raycast + block list, UpdateOccupancyVoxelFunctor, projective_occupancy_integrator_impl.cuh:27-73) and
 * nvb_mapper_update_esdf runs EsdfIntegrator::integrateBlocks(OccupancyLayer, ...) (esdf_integrator.h:72-80). */
NVB_API void nvb_default_occupancy_params(NvbOccupancyParams* p);
NVB_API int32_t nvb_mapper_set_occupancy_params(NvbMapper* m, const NvbOccupancyParams* p);
NVB_API int32_t nvb_mapper_get_occupancy_params(const NvbMapper* m, NvbOccupancyParams* p);

/* TsdfDecayIntegrator / OccupancyDecayIntegrator parameters (C/include/nvblox/integrators/tsdf_decay_integrator_params.h:21-48,
 * occupancy_decay_integrator_params.h:21-43, internal/decay_integrator_base_params.h:22-29; setters
 * tsdf_decay_integrator.h:73-101, occupancy_decay_integrator.h:72-101). */
typedef struct NvbTsdfDecayParams {
  float decay_factor;                   /* 0.95: weight *= decay_factor                                  */
  float decayed_weight_threshold;       /* 1e-3: weights never decay below it; below = "fully decayed" */
  int32_t set_free_distance_on_decayed; /* 0                                                            */
  float free_distance_vox;              /* 4                                                            */
  int32_t deallocate_decayed_blocks;    /* 1: blocks whose voxels are all fully decayed leave the map   */
} NvbTsdfDecayParams;
typedef struct NvbOccupancyDecayParams {
  float free_region_decay_probability;     /* 0.55, in [0.5, 1]  */
  float occupied_region_decay_probability; /* 0.4, in [0, 0.5)   */
  float decay_to_probability;              /* 0.5 (decay_to_free(true): 0.49, occupancy_decay_integrator.h:35-36) */
  int32_t deallocate_decayed_blocks;       /* 1                  */
} NvbOccupancyDecayParams;
/* DecayBlockExclusionOptions (C/include/nvblox/integrators/internal/decayer.h:31-44): blocks that are spared. */
typedef struct NvbDecayExclusion {
  const int32_t* excluded_blocks_xyz_host; /* may be NULL when the count is 0; a negative count is NVB_ERR_INVALID_ARGUMENT */
  int32_t num_excluded_blocks;
  int32_t has_exclusion_sphere;            /* blocks whose origin is within the sphere are spared */
  float exclusion_center[3];
  float exclusion_radius_m;
} NvbDecayExclusion;
NVB_API void nvb_default_tsdf_decay_params(NvbTsdfDecayParams* p);
NVB_API int32_t nvb_mapper_set_tsdf_decay_params(NvbMapper* m, const NvbTsdfDecayParams* p);
NVB_API int32_t nvb_mapper_get_tsdf_decay_params(const NvbMapper* m, NvbTsdfDecayParams* p);
NVB_API void nvb_default_occupancy_decay_params(NvbOccupancyDecayParams* p);
NVB_API int32_t nvb_mapper_set_occupancy_decay_params(NvbMapper* m, const NvbOccupancyDecayParams* p);
NVB_API int32_t nvb_mapper_get_occupancy_decay_params(const NvbMapper* m, NvbOccupancyDecayParams* p);
/* The constant-z slice of the 2-D ESDF (esdf_slice_min_height / esdf_slice_max_height / esdf_slice_height,
 * C/include/nvblox/integrators/esdf_integrator_params.h:33-43; setters esdf_integrator.h:216-256). */
typedef struct NvbEsdfSliceParams {
  float slice_min_height_m; /* 0 */
  float slice_max_height_m; /* 1 */
  float slice_height_m;     /* 1: z of the output slice */
  /* planar slices (slice_height_above_plane_m / slice_height_thickness_m, esdf_integrator_params.h:45-52) */
  float slice_height_above_plane_m; /* 0   */
  float slice_height_thickness_m;   /* 0.1 */
} NvbEsdfSliceParams;
NVB_API void nvb_default_esdf_slice_params(NvbEsdfSliceParams* p);
NVB_API int32_t nvb_mapper_set_esdf_slice_params(NvbMapper* m, const NvbEsdfSliceParams* p);
NVB_API int32_t nvb_mapper_get_esdf_slice_params(const NvbMapper* m, NvbEsdfSliceParams* p);

/* FreespaceIntegrator parameters (C/include/nvblox/integrators/freespace_integrator_params.h:22-58; setters
 * freespace_integrator.h:75-128). */
typedef struct NvbFreespaceParams {
  float max_tsdf_distance_for_occupancy_m;                 /* 0.15 */
  int64_t max_unobserved_to_keep_consecutive_occupancy_ms; /* 200  */
  int64_t min_duration_since_occupied_for_freespace_ms;    /* 1000 */
  int64_t min_consecutive_occupancy_duration_for_reset_ms; /* 2000 */
  int32_t check_neighborhood;                              /* 1    */
  int32_t initialize_to_high_confidence_freespace;         /* 0    */
} NvbFreespaceParams;
NVB_API void nvb_default_freespace_params(NvbFreespaceParams* p);
NVB_API int32_t nvb_mapper_set_freespace_params(NvbMapper* m, const NvbFreespaceParams* p);
NVB_API int32_t nvb_mapper_get_freespace_params(const NvbMapper* m, NvbFreespaceParams* p);
NVB_API float nvb_mapper_voxel_size(const NvbMapper* m);
NVB_API float nvb_mapper_block_size(const NvbMapper* m);

/* ViewCalculator::getBlocksInImageViewRaycast<Camera> (view_calculator.h:75-80,
 * view_calculator_impl.cuh:117-198). Does not touch the map. Writes up to
 * cap triples to out_xyz_host (x-fastest order inside the view AABB) and the
 * full count to *out_count. */
NVB_API int32_t nvb_view_raycast(NvbMapper* m, const float* depth, int32_t depth_memory,
                                 int32_t rows, int32_t cols, const float* T_L_C,
                                 const NvbCamera* cam, float block_size,
                                 float max_integration_distance_behind_surface_m,
                                 float max_integration_distance_m, int32_t* out_xyz_host,
                                 int32_t cap, int32_t* out_count);

/* Mapper::markUnobservedTsdfFreeInsideRadius(center, radius) (C/include/nvblox/mapper/mapper.h:352-356, src/mapper/mapper.cpp:494-507)
 * = Projective{Tsdf,Occupancy}Integrator::markUnobservedFreeInsideRadius (projective_integrator_impl.cuh:408-462): every block
 * whose box is closer than `radius` to `center` is allocated in the projective layer and its unobserved voxels are set to
 * slightly observed free space (TSDF: truncation distance, weight 0.1 where weight < 1e-3; occupancy: log odds -2e-4 where
 * |log odds| < 1e-4); the blocks join the tracker, so the next ESDF update covers them. updated_xyz_host may be NULL; it receives up to cap triples (unordered). */
NVB_API int32_t nvb_mapper_mark_unobserved_free_inside_radius(NvbMapper* m, const float center[3], float radius,
                                                              int32_t* updated_xyz_host, int32_t cap, int32_t* out_count);

/* ProjectiveColorIntegrator's parameters (C/include/nvblox/integrators/projective_appearance_integrator.h:96-175,
 * projective_integrator_params.h:24-75), with those of its SphereTracer (rays/sphere_tracer.h:204-218) and of its own
 * ViewCalculator's workspace bounds. sphere_tracer_maximum_ray_length_m is a separate field because the reference
 * copies max_integration_distance_m into the tracer in the constructor only
 * (src/integrators/projective_appearance_integrator.cu:61). */
typedef struct {
  float max_integration_distance_m;                 /* 7.0 */
  float truncation_distance_vox;                    /* 4.0 */
  float max_weight;                                 /* 5.0 */
  float measurement_weight;                         /* 0.8, in (0, 1] */
  int32_t sphere_tracing_ray_subsampling_factor;    /* 4; must divide the image size */
  int32_t sphere_tracer_maximum_steps;              /* 100 */
  float sphere_tracer_maximum_ray_length_m;         /* 7.0 */
  float sphere_tracer_surface_distance_epsilon_vox; /* 0.1 */
  int32_t workspace_bounds_type;                    /* NVB_WS_UNBOUNDED */
  float workspace_min[3], workspace_max[3];
} NvbColorParams;
NVB_API void nvb_default_color_params(NvbColorParams* p);
NVB_API int32_t nvb_mapper_set_color_params(NvbMapper* m, const NvbColorParams* p);
NVB_API int32_t nvb_mapper_get_color_params(const NvbMapper* m, NvbColorParams* p);

/* Mapper::integrateColor(MaskedColorImageConstView, T_L_C, Camera) (mapper.h:202-207, mapper_impl.h:104-130) =
 * ProjectiveColorIntegrator::integrateFrame (src/integrators/projective_appearance_integrator.cu:68-165): the TSDF blocks
 * in the camera's view (ViewCalculator::getBlocksInImageViewProjection) that touch the truncation band get a colour block;
 * a sphere-traced synthetic depth image of the TSDF layer (SphereTracer::renderImageOnGPU) decides occlusion; visible voxels
 * blend the bilinearly interpolated pixel in (UpdateAppearanceVoxelFunctor). color = rows * cols * 3 bytes, RGB, row-major;
 * mask (rows * cols, may be NULL) and mask_mode as for depth. With an occupancy mapper the call does nothing, as in the
 * reference. updated_xyz_host may be NULL; otherwise it receives up to cap triples of `updated_blocks` (unordered) and
 * *out_count the full count. */
NVB_API int32_t nvb_mapper_integrate_color(NvbMapper* m, const uint8_t* color, const uint8_t* mask, int32_t mask_mode,
                                           int32_t memory, int32_t rows, int32_t cols, const float* T_L_C,
                                           const NvbCamera* cam, int32_t* updated_xyz_host, int32_t cap, int32_t* out_count);
/* A call with device-resident images (memory = NVB_MEM_DEVICE) and no output pointers is enqueued without synchronising;
 * after nvb_mapper_synchronize, this returns the `updated_blocks` of the last colour frame. */
NVB_API int32_t nvb_mapper_last_color_blocks(NvbMapper* m, int32_t* out_xyz_host, int32_t cap, int32_t* out_count);
/* SphereTracer::renderImageOnGPU(camera, T_L_C, tsdf_layer, truncation_distance_m, &depth, ..., ray_subsampling_factor)
 * (C/src/rays/sphere_tracer.cu:389-485) with the colour integrator's tracer settings: out_depth_host receives
 * (height / f) * (width / f) floats, -1 where a ray found no surface. */
NVB_API int32_t nvb_sphere_tracer_render_depth(NvbMapper* m, const float* T_L_C, const NvbCamera* cam,
                                               float truncation_distance_m, int32_t ray_subsampling_factor,
                                               float* out_depth_host);

/* A standalone SphereTracer's parameters (C/include/nvblox/rays/sphere_tracer.h:204-218); each must be positive
 * (the setters' CHECK_GTs, C/src/rays/sphere_tracer.cu:319-333). */
typedef struct {
  int32_t maximum_steps;              /* 100 */
  float maximum_ray_length_m;         /* 15.0 */
  float surface_distance_epsilon_vox; /* 0.1 */
} NvbSphereTracerParams;
NVB_API void nvb_default_sphere_tracer_params(NvbSphereTracerParams* p);
/* SphereTracer::renderImageOnGPU(camera, T_L_C, tsdf_layer, truncation_distance_m, &depth, memory, ray_subsampling_factor)
 * (C/src/rays/sphere_tracer.cu:134-173, 389-485) of the mapper's TSDF layer: out_depth receives (height / f) * (width / f)
 * floats, row-major, the depth t * d_C.z of each converged ray and -1 elsewhere. Ray (r, c) goes through the image-plane
 * point f * (c, r) + f / 2. f must divide the image size; an occupancy mapper has no TSDF layer to trace.
 * memory = NVB_MEM_DEVICE: the render is enqueued on `stream` (a cudaStream_t; NULL is the default stream) after the work
 * already there and on the mapper, the stream's next work and the mapper's follow it, and nothing synchronises.
 * memory = NVB_MEM_HOST: the outputs are staged on the device and written when the call returns. */
NVB_API int32_t nvb_render_depth(NvbMapper* m, const NvbSphereTracerParams* p, const float* T_L_C, const NvbCamera* cam,
                                 float truncation_distance_m, int32_t ray_subsampling_factor, int32_t memory, float* out_depth,
                                 void* stream);
/* SphereTracer::renderRgbdImageOnGPU (C/src/rays/sphere_tracer.cu:239-300, 487-644): the depth of nvb_render_depth, and in
 * out_rgb 3 bytes (r, g, b) per ray: the colour of the colour voxel that holds the hit point T_L_C.t + t * d_L, whatever its
 * weight (an allocated block that was never coloured gives grey 127). A miss, a hit without a colour block, and every hit of
 * a mapper that never integrated colour, give black. Memory and ordering as nvb_render_depth. */
NVB_API int32_t nvb_render_rgbd(NvbMapper* m, const NvbSphereTracerParams* p, const float* T_L_C, const NvbCamera* cam,
                                float truncation_distance_m, int32_t ray_subsampling_factor, int32_t memory, float* out_depth,
                                uint8_t* out_rgb, void* stream);

/* primitives::Scene (C/include/nvblox/primitives/primitives.h, scene.h, src/primitives/primitives.cpp, scene.cpp,
 * primitives/internal/impl/scene_impl.h): planes, cubes, spheres and cylinders, and the exact distance fields and depth images
 * they give. Primitive::Type order. */
typedef enum { NVB_PRIM_PLANE = 0, NVB_PRIM_CUBE = 1, NVB_PRIM_SPHERE = 2, NVB_PRIM_CYLINDER = 3 } NvbPrimitiveType;
/* One primitive: params are the plane's unit normal (norm 1 +- 1e-3), the cube's x, y, z size, the sphere's radius, or the
 * cylinder's radius and height (axis along z); the unused entries are ignored. */
typedef struct {
  int32_t type;
  float center[3];
  float params[4];
} NvbPrimitive;
/* A scene: the primitives (host memory, any number) and the box a generated layer covers (Scene::aabb(), by default
 * (-5, -5, -1) to (5, 5, 9)). */
typedef struct {
  const NvbPrimitive* primitives;
  int32_t num_primitives;
  float aabb_min[3];
  float aabb_max[3];
} NvbScene;
/* Scene::generateDepthImageFromScene(camera, T_S_C, max_dist, &depth, invalid_depth): out_depth receives height * width
 * floats, row-major; pixel (r, c) casts the ray T_S_C.linear() * vectorFromPixelIndices((c, r)).normalized() from T_S_C's
 * origin, and gets the z of the nearest hit within max_dist in the camera frame, or invalid_depth.
 * memory = NVB_MEM_DEVICE: enqueued on `stream` (a cudaStream_t on the current device; NULL is the default stream), nothing
 * synchronises. memory = NVB_MEM_HOST: the image is written when the call returns. */
NVB_API int32_t nvb_scene_render_depth(const NvbScene* scene, const NvbCamera* cam, const float* T_S_C, float max_dist,
                                       float invalid_depth, int32_t memory, float* out_depth, void* stream);
/* Scene::getSignedDistanceToPoint(p, max_dist) of n points (xyz, 3 floats each) into out (n floats); both in `memory`,
 * ordered like nvb_scene_render_depth. */
NVB_API int32_t nvb_scene_signed_distance(const NvbScene* scene, const float* xyz, int32_t memory, int64_t n, float max_dist,
                                          float* out, void* stream);
/* Scene::generateLayerFromScene<VoxelType>(max_dist, layer) on the mapper's layer_id: NVB_LAYER_TSDF or NVB_LAYER_OCCUPANCY
 * (whichever is the mapper's projective layer) or NVB_LAYER_FREESPACE (a mapper with one). Every block the AABB touches is
 * allocated; then every voxel of the layer whose centre lies in the (closed) AABB is written: TSDF max(sdf, -max_dist) with
 * weight 1, occupancy the log odds of probability 1 where sdf <= sqrt(3) * voxel_size / 2 and of 0 elsewhere, freespace only
 * is_high_confidence_freespace, true where sdf is above that. The block-update tracker is not told. An AABB of more than
 * 2^28 blocks is NVB_ERR_CAPACITY and changes nothing. Synchronous. */
NVB_API int32_t nvb_scene_generate_layer(NvbMapper* m, int32_t layer_id, const NvbScene* scene, float max_dist);
/* nvblox_torch's Scene::toMapper for one mapper (nvblox_torch/cpp/src/py_scene.cu): the projective layer (TSDF, or
 * occupancy on an occupancy mapper) is replaced by the scene's layer with max_dist = 4 voxels, like VoxelBlockLayer::copyFrom;
 * every block of it is marked for the ESDF, freespace and mesh consumers, and the ESDF is updated. The colour, mesh and
 * freespace layers are left as they are. Synchronous. */
NVB_API int32_t nvb_scene_to_mapper(NvbMapper* m, const NvbScene* scene);

/* Mapper::integrateDepth(MaskedDepthImageConstView, T_L_C, Camera)
 * (mapper.h:167-172, mapper_impl.h:28-81) =
 * ProjectiveTsdfIntegrator::integrateFrame (projective_tsdf_integrator.h:48-52)
 * + BlocksToUpdateTracker::addBlocksToUpdate. mask may be NULL
 * (kMaskActiveEverywhere). updated_xyz_host may be NULL; otherwise it receives
 * up to cap triples of `updated_blocks` and *out_count the full count. */
NVB_API int32_t nvb_mapper_integrate_depth(NvbMapper* m, const float* depth, const uint8_t* mask,
                                           int32_t mask_mode, int32_t memory, int32_t rows,
                                           int32_t cols, const float* T_L_C, const NvbCamera* cam,
                                           int32_t* updated_xyz_host, int32_t cap,
                                           int32_t* out_count);

/* Same work, enqueued on the mapper's stream; returns without synchronising.
 * Host depth/mask buffers must stay valid (and should be pinned) until
 * nvb_mapper_synchronize. The per-frame block count can be read afterwards with
 * nvb_mapper_last_frame_block_count. */
NVB_API int32_t nvb_mapper_integrate_depth_async(NvbMapper* m, const float* depth,
                                                 const uint8_t* mask, int32_t mask_mode,
                                                 int32_t memory, int32_t rows, int32_t cols,
                                                 const float* T_L_C, const NvbCamera* cam);

/* Mapper::updateEsdf(UpdateFullLayer) (mapper.h:326, src/mapper/mapper.cpp:408-430):
 * EsdfIntegrator::integrateBlocks over the blocks touched since the last call
 * (all TSDF blocks on the first call or when update_full_layer != 0). */
NVB_API int32_t nvb_mapper_update_esdf(NvbMapper* m, int32_t update_full_layer);
NVB_API int32_t nvb_mapper_update_esdf_async(NvbMapper* m, int32_t update_full_layer);

/* Mapper::decayTsdf / decayOccupancy (mapper.h:268-292; mapper_impl.h:190-265; VoxelDecayer::decay,
 * C/include/nvblox/integrators/internal/cuda/impl/decayer_impl.cuh:150-262) on the mapper's projective layer.
 * depth == NULL: decay*AllVoxels. depth != NULL: decay*ExcludeLastView -- voxels that have a depth measurement in
 * the given view (doesVoxelHaveDepthMeasurement, projective_integrators_common_impl.cuh:58-101, with the
 * integrator's max integration distance and truncation distance) are spared; the caller passes the view it wants
 * excluded (the reference's Mapper keeps a copy of the last frame for this). `exclusion` (may be NULL) spares whole
 * blocks. Fully decayed blocks are deallocated when the parameters say so, from the projective AND the ESDF
 * layer (Mapper::clearBlocksInLayers, src/mapper/mapper.cpp:546-575), their indices are written to
 * removed_xyz_host (up to cap; may be NULL) and counted in *out_count; the next nvb_mapper_update_esdf covers all
 * blocks (BlocksToUpdateTracker::addAllBlocksToUpdate). Synchronous. */
NVB_API int32_t nvb_mapper_decay(NvbMapper* m, const NvbDecayExclusion* exclusion, const float* depth,
                                 int32_t depth_memory, int32_t rows, int32_t cols, const float* T_L_C,
                                 const NvbCamera* cam, int32_t* removed_xyz_host, int32_t cap, int32_t* out_count);

/* Mapper::updateFreespace(update_time_ms, T_L_C, sensor, depth_frame, update_full_layer) (mapper.h:196-214,
 * mapper_impl.h:152-188) on a NVB_PROJECTIVE_TSDF_WITH_FREESPACE mapper: FreespaceIntegrator::updateFreespaceLayer
 * (C/include/nvblox/integrators/internal/cuda/impl/freespace_integrator_impl.cuh:99-383) over the TSDF blocks touched
 * since the last call (all on the first call / update_full_layer). depth != NULL: only voxels with a depth measurement
 * in that view are updated (max view distance = the integrator's max integration distance, truncation = 2 x the
 * truncation distance, mapper_impl.h:157-172); depth == NULL: no viewpoint exclusion. Synchronous. The following
 * nvb_mapper_update_esdf treats high-confidence-free voxels as outside (esdf_integrator.cu:401-415). */
NVB_API int32_t nvb_mapper_update_freespace(NvbMapper* m, int64_t update_time_ms, const float* depth, int32_t depth_memory,
                                            int32_t rows, int32_t cols, const float* T_L_C, const NvbCamera* cam,
                                            int32_t update_full_layer);
/* FreespaceIntegrator::updateFreespaceLayer on an explicit block list (freespace_integrator.h:60-66); max_view_distance_m
 * / truncation_distance_m <= 0 mean "unset" (no limit). Does not consult or reset the tracker. */
NVB_API int32_t nvb_freespace_update_blocks(NvbMapper* m, const int32_t* blocks_xyz_host, int32_t num_blocks,
                                            int64_t update_time_ms, const float* depth, int32_t depth_memory, int32_t rows,
                                            int32_t cols, const float* T_L_C, const NvbCamera* cam,
                                            float max_view_distance_m, float truncation_distance_m);

/* Mapper::decayTsdfExcludeLastView / decayOccupancyExcludeLastView (mapper.h:218-230) with the view the mapper kept
 * (NvbMapperOptions.keep_last_view); decays every voxel if no frame was integrated yet, like the reference. */
NVB_API int32_t nvb_mapper_decay_exclude_last_view(NvbMapper* m, const NvbDecayExclusion* exclusion,
                                                   int32_t* removed_xyz_host, int32_t cap, int32_t* out_count);

/* BoundingShape (C/include/nvblox/geometry/bounding_shape.h:26, bounding_spheres.h, bounding_boxes.h):
 * NVB_SHAPE_SPHERE: a = centre, b[0] = radius; NVB_SHAPE_AABB: a = minimum corner, b = maximum corner. */
typedef enum { NVB_SHAPE_SPHERE = 0, NVB_SHAPE_AABB = 1 } NvbShapeType;
typedef struct NvbBoundingShape {
  int32_t type; /* NvbShapeType */
  float a[3];
  float b[3];
} NvbBoundingShape;

/* Mapper::clearOutsideRadius(center, radius) (C/src/mapper/mapper.cpp:473-492): every block of the projective layer
 * whose box is farther than `radius` from `center` (exteriorDistance > radius, strict; src/geometry/bounding_spheres.cpp:
 * 23-31,47-50,69-74) is deallocated, and with it its twins (Mapper::clearBlocksInLayers, mapper.cpp:546-634): colour, mesh
 * and freespace blocks, the ESDF block (3-D) or the column's slice block when no projective block is left in the column
 * between the slice bounds (2-D). The blocks leave every initialised tracker consumer
 * (BlocksToUpdateTracker::removeClearedBlocksFromTracking, src/map/blocks_to_update_tracker.cpp:75-90) and join the
 * cleared-blocks set. The radius is not checked: radius <= 0 removes every block that does not contain the centre.
 * removed_xyz_host (may be NULL) receives up to cap removed triples in (x, y, z) order; *out_count the number removed.
 * Synchronous; waits for an ESDF update still in flight. */
NVB_API int32_t nvb_mapper_clear_outside_radius(NvbMapper* m, const float center[3], float radius, int32_t* removed_xyz_host,
                                                int32_t cap, int32_t* out_count);
/* Mapper::clearTsdfInsideShapes(shapes) (mapper.cpp:364-368): ShapeClearer<TsdfLayer>::clear on the TSDF layer, then the
 * touched blocks join every initialised tracker consumer (addBlocksToUpdate). Nothing is allocated or deallocated; on an
 * occupancy mapper (no TSDF layer) nothing happens. updated_xyz_host (may be NULL) receives up to cap touched triples in
 * (x, y, z) order; *out_count the number touched. Synchronous. */
NVB_API int32_t nvb_mapper_clear_tsdf_inside_shapes(NvbMapper* m, const NvbBoundingShape* shapes, int32_t num_shapes,
                                                    int32_t* updated_xyz_host, int32_t cap, int32_t* out_count);
/* ShapeClearer<LayerType>::clear (C/include/nvblox/integrators/internal/cuda/impl/shape_clearer_impl.cuh:22-127) on the
 * NVB_LAYER_TSDF, NVB_LAYER_OCCUPANCY or NVB_LAYER_COLOR layer: in every block a shape touches (sphere: exteriorDistance <
 * radius; box: inclusive AlignedBox::intersects), the voxels whose centre a shape contains (sphere: distance <= radius; box:
 * inclusive) are reset -- TSDF distance 0 and weight 0, occupancy log odds 0, colour Color::Gray() and weight 0. The
 * tracker is not told. Output as for nvb_mapper_clear_tsdf_inside_shapes. Synchronous. */
NVB_API int32_t nvb_layer_clear_shapes(NvbMapper* m, int32_t layer, const NvbBoundingShape* shapes, int32_t num_shapes,
                                       int32_t* updated_xyz_host, int32_t cap, int32_t* out_count);
/* Mapper::getClearedBlocks(blocks_to_ignore) (mapper.cpp:509-521): the blocks deallocated by nvb_mapper_clear_outside_radius
 * or nvb_mapper_decay since the last call, minus ignore_xyz (may be NULL when n_ignore is 0), in (x, y, z) order; the set
 * is emptied. out_xyz_host == NULL: *out_count receives the current set size and nothing changes. A set larger than cap
 * fails with NVB_ERR_CAPACITY and stays as it is (the ignored blocks removed). */
NVB_API int32_t nvb_mapper_get_cleared_blocks(NvbMapper* m, const int32_t* ignore_xyz, int32_t n_ignore, int32_t* out_xyz_host,
                                              int32_t cap, int32_t* out_count);

/* Mapper::updateEsdfSlice (mapper.h:331-343; EsdfMode::k2D) = EsdfIntegrator::integrateSlice with the constant-z
 * slice description (C/src/integrators/esdf_integrator.cu:283-347, markSitesInSlice :754-1055): the band
 * [slice_min_height, slice_max_height] of the projective layer (honouring the freespace layer if the mapper has one) is
 * squashed onto ONE layer of ESDF blocks at slice_height; clear + computeEsdf then run on that layer. A mapper's ESDF
 * layer is either 3-D or 2-D: mixing nvb_mapper_update_esdf and nvb_mapper_update_esdf_slice is an error, like the
 * reference's EsdfMode check. Synchronous. */
NVB_API int32_t nvb_mapper_update_esdf_slice(NvbMapper* m, int32_t update_full_layer);
/* The same with a PlanarSliceDescription (Mapper::updateEsdfSlice(..., ground_plane), mapper.h:343;
 * EsdfIntegrator::integrateSlice(layer, blocks, ground_plane, esdf), esdf_integrator.h:120-150): the band starts
 * slice_height_above_plane_m above the plane n . p + d = 0 and is slice_height_thickness_m thick, per voxel column
 * (PlanarSliceColumnBoundsGetter). plane = {nx, ny, nz, d} = Plane::normal() (unit length) and Plane::offset(); a
 * near-vertical plane (|nz| < 1e-4) falls back to z = 0 like checkForVerticalPlane. */
NVB_API int32_t nvb_mapper_update_esdf_slice_planar(NvbMapper* m, const float plane[4], int32_t update_full_layer);
NVB_API int32_t nvb_esdf_integrate_slice_planar_blocks(NvbMapper* m, const float plane[4], const int32_t* blocks_xyz_host,
                                                       int32_t num_blocks);
/* EsdfIntegrator::integrateSlice(layer, block_indices, esdf_layer) on an explicit block list (esdf_integrator.h:96-118). */
NVB_API int32_t nvb_esdf_integrate_slice_blocks(NvbMapper* m, const int32_t* blocks_xyz_host, int32_t num_blocks);

/* GroundPlaneEstimator (C/include/nvblox/experimental/ground_plane/ground_plane_estimator.h,
 * ground_plane_estimator_params.h, ransac_plane_fitter_params.h, tsdf_zero_crossings_extractor.h), one per mapper. */
typedef struct NvbGroundPlaneParams {
  float ground_points_candidates_min_z_m; /* -0.1: candidates keep min_z <= z <= max_z */
  float ground_points_candidates_max_z_m; /* 0.15 */
  float ransac_distance_threshold_m;      /* 0.2: MSAC inlier threshold t */
  int32_t num_ransac_iterations;          /* 1000, >= 1 */
  float min_tsdf_weight;                  /* 0.1: both voxels of a crossing need weight >= this */
  int32_t max_crossings;                  /* 360000: a layer with this many crossings or more gives no plane */
} NvbGroundPlaneParams;
NVB_API void nvb_default_ground_plane_params(NvbGroundPlaneParams* p);
NVB_API int32_t nvb_mapper_set_ground_plane_params(NvbMapper* m, const NvbGroundPlaneParams* p);
NVB_API int32_t nvb_mapper_get_ground_plane_params(const NvbMapper* m, NvbGroundPlaneParams* p);
/* GroundPlaneEstimator::computeGroundPlane(tsdf_layer) (ground_plane_estimator.cpp:27-62):
 *   1. the zero crossings from above of the TSDF layer (computeZeroCrossingsFromAboveOnGPU): every voxel pair (v, v + z)
 *      with both weights >= min_tsdf_weight, distance(v + z) > 0 and distance(v) <= 0 gives the point
 *      centre(v) + (0, 0, -d(v) * voxel_size / (d(v + z) - d(v))); pairs whose upper voxel lies in a missing block are
 *      skipped. The list is in canonical order: block index (x, y, z) lexicographically, then voxel (x, y, z);
 *   2. the ground candidates: the finite crossings with min_z <= z <= max_z, in the same order;
 *   3. the MSAC plane of the candidates (as nvb_ransac_fit_plane).
 * *found = 0 when the layer has no blocks, the mapper has no TSDF layer (occupancy), the crossings number max_crossings or
 * more, fewer than 3 candidates remain or no sample gives a plane; the estimator's last crossings, candidates and plane are
 * then cleared (resetInternal). Otherwise plane = {nx, ny, nz, d} (unit normal, n . p + d = 0) and all three are kept.
 * Synchronous: reads back the two counts and the 20-byte result only. */
NVB_API int32_t nvb_mapper_compute_ground_plane(NvbMapper* m, float plane[4], int32_t* found);
/* GroundPlaneEstimator::ground_plane(): the plane of the last computeGroundPlane, *found = 0 if there is none. */
NVB_API int32_t nvb_mapper_ground_plane(NvbMapper* m, float plane[4], int32_t* found);
typedef enum { NVB_GROUND_POINTS_CROSSINGS = 0, NVB_GROUND_POINTS_CANDIDATES = 1 } NvbGroundPoints;
/* tsdf_zero_crossings() / tsdf_zero_crossings_ground_candidates() of the last computeGroundPlane: *valid = 0 if there are
 * none (never computed or cleared by a failure); else *n = the number of points and up to cap of them are written to
 * xyz (x, y, z floats; may be NULL) in the canonical order. */
NVB_API int32_t nvb_mapper_ground_plane_points(NvbMapper* m, int32_t which, float* xyz, int32_t cap, int32_t* n, int32_t* valid);
/* RansacPlaneFitter::fit (ransac_plane_fitter.cu:29-144), MSAC: iteration i draws three indices curand() % n from the
 * XORWOW state curand_init(1234, i, 0), builds Plane::planeFromPoints (rejects equal or collinear samples) and sums, over
 * the points in order and in float, d^2 if |d| < threshold else threshold^2. The lowest cost wins (lowest iteration on
 * ties). *found = 0 for n < 3 or when every sample is rejected. points: n x 3 floats on the host or the device (memory).
 * Uses the mapper's device, stream and cached generator states; the estimator's state is not touched. Synchronous. */
NVB_API int32_t nvb_ransac_fit_plane(NvbMapper* m, const float* points, int32_t memory, int32_t n, int32_t num_ransac_iterations,
                                     float ransac_distance_threshold_m, float plane[4], int32_t* found);

/* DynamicsDetection::computeDynamics(depth, freespace_layer, camera, T_L_C) (C/include/nvblox/dynamics/dynamics_detection.h,
 * dynamics/internal/cuda/impl/dynamics_detection_impl.cuh:26-130) on the freespace layer of a
 * NVB_PROJECTIVE_TSDF_WITH_FREESPACE mapper (NVB_ERR_INVALID_ARGUMENT on any other), as that layer stands. A pixel with
 * depth > 0 (NaN included) whose point T_L_C * unproject(pixel, depth) falls into an allocated freespace voxel that is
 * high-confidence freespace is dynamic: mask 255 and overlay (255, s, s), s = min(25.5 * depth, 255); other looked-up
 * pixels get mask 0 and (0, s, s); the rest mask 0 and white. The dynamic points come in row-major pixel order (the
 * reference's order is an atomicAdd race). Host depth is staged in a buffer the mapper keeps. The call is enqueued on
 * the mapper's stream without a host synchronisation; the point count stays on the device until a getter asks. */
NVB_API int32_t nvb_mapper_compute_dynamics(NvbMapper* m, const float* depth, int32_t memory, int32_t rows, int32_t cols,
                                            const float* T_L_C, const NvbCamera* cam);
/* MaskPreprocessor::removeSmallConnectedComponents(mask_in, threshold, mask_out) (C/src/sensors/mask_preprocessor.cpp:
 * 140-183): threshold <= 0 copies the mask. Otherwise the mask is downscaled by 2 (pixel (2r, 2c)), its pixels > 0 are
 * labelled into 4-connected components, components of fewer than threshold / 4 (integer division) downscaled pixels are
 * erased, survivors hold 254, and the result is upscaled by 2. Unlike the reference, whose output shrinks to
 * (rows / 2) * 2 x (cols / 2) * 2, mask_out keeps the input's size: a trailing odd row or column is 0. Both masks are
 * rows x cols bytes in `memory`; they may be the same buffer. Runs on the mapper's stream with its scratch; with device
 * masks it does not synchronise, with host masks it returns when mask_out is written. */
NVB_API int32_t nvb_mapper_remove_small_components(NvbMapper* m, const uint8_t* mask_in, uint8_t* mask_out, int32_t memory,
                                                   int32_t rows, int32_t cols, int32_t threshold);
/* DynamicsDetection::getDynamicMaskImage / getDynamicOverlayImage of the last nvb_mapper_compute_dynamics: *rows, *cols of
 * the frame (0 x 0 before the first call); out (rows x cols bytes, resp. x 3 for the RGB overlay, in `memory`) may be NULL.
 * A host copy synchronises the mapper's stream; a device copy is enqueued on it. */
NVB_API int32_t nvb_mapper_dynamic_mask(NvbMapper* m, uint8_t* out, int32_t memory, int32_t* rows, int32_t* cols);
NVB_API int32_t nvb_mapper_dynamic_overlay(NvbMapper* m, uint8_t* out, int32_t memory, int32_t* rows, int32_t* cols);
/* DynamicsDetection::getDynamicPointsHost / getDynamicPointcloudDevice: *out_count = the number of dynamic points of the
 * last frame (read back here: this synchronises the mapper's stream), and the first min(count, cap) of them (x, y, z
 * floats) are copied to xyz (in `memory`; may be NULL). */
NVB_API int32_t nvb_mapper_dynamic_points(NvbMapper* m, float* xyz, int32_t memory, int32_t cap, int32_t* out_count);
/* The detector's device buffers, for a consumer on another stream (a second mapper, through nvb_mapper_wait_for). They
 * stay valid, and their contents unchanged, until the next nvb_mapper_compute_dynamics on this mapper or its destruction.
 * cleaned_mask is a rows x cols buffer kept for nvb_mapper_remove_small_components' output. */
typedef struct {
  const float* depth;           /* the last frame's depth, staged on the device */
  const uint8_t* mask;          /* the dynamic mask */
  uint8_t* cleaned_mask;        /* scratch of the same size, for the filtered mask */
  const uint8_t* overlay;       /* RGB */
  const float* points;          /* x, y, z per dynamic point */
  const int32_t* num_points;    /* device */
  int32_t rows, cols;
} NvbDynamicsBuffers;
NVB_API int32_t nvb_mapper_dynamics_device_buffers(NvbMapper* m, NvbDynamicsBuffers* out);
/* Device-side ordering between two mappers: work enqueued on waiter's stream after this call runs after everything
 * enqueued so far on producer's stream. No host synchronisation. */
NVB_API int32_t nvb_mapper_wait_for(NvbMapper* waiter, NvbMapper* producer);

/* ImageMasker parameters (C/include/nvblox/semantics/image_masker.h:110-119). */
typedef struct {
  float occlusion_threshold_m;              /* 0.25: a point more than this behind the nearest one seen from the mask camera is occluded */
  float depth_masked_image_invalid_pixel;   /* -1: written to the masked (foreground) output where the pixel is not masked */
  float depth_unmasked_image_invalid_pixel; /* -1: written to the unmasked (background) output where the pixel is masked */
} NvbImageMaskerParams;
NVB_API void nvb_default_image_masker_params(NvbImageMaskerParams* p);
/* ImageMasker::splitImageOnGPU(depth, mask, T_CM_CD, depth_camera, mask_camera, ...) (C/src/semantics/image_masker.cu:
 * 316-392) in three launches on the mapper's stream: a mask-sized min-depth image is filled with FLT_MAX; every depth pixel
 * is unprojected, moved by T_CM_CD (column-major 4x4) into the mask camera and projected, and its z is min-reduced into
 * the 5 x 5 patch around (int)(u + k - 2), (int)(v + k - 2); then a pixel goes to the foreground when it projects, the mask
 * (bytes != 0) is set at (int)u, (int)v and min_depth + occlusion_threshold_m >= z there. Every other pixel, and every +-inf
 * or NaN depth, goes to the background. Each output holds the depth where the other holds its invalid value. With
 * with_overlay != 0 the RGB overlay is grey 12.75 * depth (clamped to 0..255; NaN 255) with red 255 on foreground pixels.
 * Deviations from the reference: a projection exactly on u == width or v == height is a miss here (the reference reads
 * past the mask's row); a negative depth has grey 0 (undefined in the reference). Sizes must match the cameras
 * (width x height); depth, mask (mask_rows x mask_cols bytes) are in `memory`. Host inputs are copied to the device on the
 * mapper's stream before the call returns. The outputs stay in the mapper (nvb_mapper_split_output, nvb_mapper_split_device_buffers); the call does
 * not synchronise (the reference does). */
NVB_API int32_t nvb_mapper_split_depth_image(NvbMapper* m, const float* depth, int32_t depth_rows, int32_t depth_cols,
                                             const uint8_t* mask, int32_t mask_rows, int32_t mask_cols, int32_t memory,
                                             const float* T_CM_CD, const NvbCamera* depth_cam, const NvbCamera* mask_cam,
                                             const NvbImageMaskerParams* params, int32_t with_overlay);
/* Outputs of nvb_mapper_split_depth_image. */
typedef enum { NVB_SPLIT_BACKGROUND = 0, NVB_SPLIT_FOREGROUND = 1, NVB_SPLIT_OVERLAY = 2 } NvbSplitOutput;
/* One output of the last split: *rows, *cols of the frame (0 x 0 before the first split, and for the overlay when the last
 * split made none); out (rows x cols floats, resp. x 3 bytes for the overlay, in `memory`) may be NULL. A host copy
 * synchronises the mapper's stream; a device copy is enqueued on it. */
NVB_API int32_t nvb_mapper_split_output(NvbMapper* m, int32_t which, void* out, int32_t memory, int32_t* rows, int32_t* cols);
/* The split's device buffers, for a consumer on another stream (a second mapper, through nvb_mapper_wait_for). They stay
 * valid, and their contents unchanged, until the next nvb_mapper_split_depth_image on this mapper or its destruction. */
typedef struct {
  const float* background;  /* the unmasked depth */
  const float* foreground;  /* the masked depth */
  const uint8_t* overlay;   /* RGB; NULL when the last split made none */
  int32_t rows, cols;
} NvbSplitBuffers;
NVB_API int32_t nvb_mapper_split_device_buffers(NvbMapper* m, NvbSplitBuffers* out);
/* ImageMasker::splitImageOnGPU(color, mask, ...) (C/src/semantics/image_masker.cu:44-78,305-314): the mask lies on top of
 * the image; a pixel with mask != 0 is copied to masked_out, the others to unmasked_out, and the other output is black.
 * overlay_out (may be NULL) is the input with red = 255 on masked pixels. rgb and the outputs are rows x cols x 3 bytes,
 * mask rows x cols bytes, all in `memory`. Device buffers: enqueued on the mapper's stream; host buffers: returns when the
 * outputs are written. */
NVB_API int32_t nvb_mapper_split_color_image(NvbMapper* m, const uint8_t* rgb, const uint8_t* mask, int32_t memory,
                                             int32_t rows, int32_t cols, uint8_t* unmasked_out, uint8_t* masked_out,
                                             uint8_t* overlay_out);

/* EsdfSlicer::sliceLayerToDistanceImage (C/include/nvblox/integrators/esdf_slicer.h:52-78, C/src/integrators/esdf_slicer.cu:
 * 25-67,112-215) and, if grid_host != NULL, EsdfSlicer::occupancyGridFromSliceImage (:78-110,254-300) of the ESDF layer
 * (3-D or 2-D) at slice_height_m: one pixel per voxel over the AABB of the ESDF blocks at that height, rows along y,
 * columns along x; value = distance in metres (negative inside), `unobserved_value` where nothing is known; grid = 100
 * occupied (distance < 0.01), 0 free, -1 unknown. Writes the AABB (min xyz, max xyz), the image size, and up to
 * cap_pixels pixels into the host buffers (either may be NULL to query the size). rows = cols = 0 if the layer has no
 * block at that height. */
NVB_API int32_t nvb_esdf_slice_distance_image(NvbMapper* m, float slice_height_m, float unobserved_value,
                                              float aabb_out[6], float* image_host, int8_t* grid_host, int32_t cap_pixels,
                                              int32_t* rows_out, int32_t* cols_out);
/* voxelLayerToDenseVoxelGridInAABBAsync (C/include/nvblox/map/internal/cuda/impl/layer_to_3d_grid_impl.cuh) on the ESDF
 * layer with the conversion of nvblox_ros's EsdfAndGradients service (R/nvblox_ros/src/lib/conversions/
 * esdf_and_gradients_conversions.cu:28-47): the voxel grid of aabb = {min xyz, max xyz} (metres; robustFloor of each corner over
 * the voxel size, both ends included), one float per voxel in z-fastest order (x slowest), the distance in metres (negative
 * inside), default_value where the voxel is unobserved or its block is not allocated. Writes the grid's first voxel index and its
 * size in voxels; the cells only if out != NULL and cap >= their number, into `memory` (NVB_MEM_HOST or NVB_MEM_DEVICE; device
 * output is complete at return). An empty box gives dims = 0. This is how the ESDF's device blocks are read as a dense grid: they
 * are not EsdfVoxel arrays (see nvb_layer_block_device_ptr). */
NVB_API int32_t nvb_esdf_dense_grid_in_aabb(NvbMapper* m, const float aabb[6], float default_value, int32_t memory, float* out,
                                            int64_t cap, int32_t min_index_out[3], int32_t dims_out[3]);
/* EsdfSlicer::getAabbOfLayerAtHeight (C/src/integrators/esdf_slicer.cu:112-147): the box of the ESDF blocks at the slice's z
 * index; *empty_out = 1 (aabb_out untouched) if there is none. */
NVB_API int32_t nvb_esdf_slice_aabb(NvbMapper* m, float slice_height_m, float aabb_out[6], int32_t* empty_out);
/* EsdfSlicer::sliceLayerToDistanceImage(layer, slice_height, unobserved_value, aabb, image) on a GIVEN box (:169-199): the
 * building block of sliceLayersToCombinedDistanceImage (C/include/nvblox/integrators/esdf_slicer.h:78-118, esdf_slicer.cu:
 * 201-240), which slices two layers (two mappers here) on the merged box of their slices and takes the element-wise minimum. */
NVB_API int32_t nvb_esdf_slice_distance_image_in_aabb(NvbMapper* m, float slice_height_m, float unobserved_value, const float aabb[6],
                                                      float* image_host, int8_t* grid_host, int32_t cap_pixels, int32_t* rows_out,
                                                      int32_t* cols_out);

/* EsdfIntegrator::integrateBlocks(const TsdfLayer&, const std::vector<Index3D>&, EsdfLayer*)
 * (esdf_integrator.h:56-58, src/integrators/esdf_integrator.cu:220-266) on an
 * explicit block list; does not consult or reset the tracker. */
NVB_API int32_t nvb_esdf_integrate_blocks(NvbMapper* m, const int32_t* blocks_xyz_host,
                                          int32_t num_blocks);

/* cudaStreamSynchronize on the mapper's stream + deferred error check. */
NVB_API int32_t nvb_mapper_synchronize(NvbMapper* m);
NVB_API int32_t nvb_mapper_last_frame_block_count(NvbMapper* m, int32_t* out_count);
/* `updated_blocks` of the most recent frame again (e.g. after a too-small buffer). */
NVB_API int32_t nvb_mapper_last_frame_blocks(NvbMapper* m, int32_t* out_xyz_host, int32_t cap,
                                             int32_t* out_count);
/* Multi-GPU merge step (no reference counterpart: the reference is single-GPU; SURVEY.md 8e): sorted unique
 * union of block-index lists. xyz_dev holds n int32 triples in device memory (e.g. the NCCL all-gather of the
 * ranks' padded lists; a triple whose x is INT32_MIN is padding), aabb_min/max bound the union. Writes up to cap
 * triples to out_xyz_dev in the view calculator's order (x fastest, then y, then z) and the count to the host. */
NVB_API int32_t nvb_blocks_union(NvbMapper* m, const int32_t* xyz_dev, int32_t n, const int32_t aabb_min[3],
                                 const int32_t aabb_max[3], int32_t* out_xyz_dev, int32_t cap,
                                 int32_t* out_count_host);

/* ViewCalculator::cache_last_viewpoint (C/include/nvblox/integrators/view_calculator.h:196; C/src/integrators/view_calculator.cu:82-88),
 * on by default like in the reference: nvb_mapper_integrate_depth* reuses the block list of one of the last two frames whose
 * pose (1 mm, 0.1 degree) and sensor match -- whatever the depth image holds (ViewpointCache, view_calculator.h:211-244). */
NVB_API int32_t nvb_mapper_set_cache_last_viewpoint(NvbMapper* m, int32_t enable);
NVB_API int32_t nvb_mapper_get_cache_last_viewpoint(const NvbMapper* m);

/* Scheduling knob with no counterpart in the reference: the cooperative ESDF wavefront launches num_SMs - reserved_sms CTAs
 * (default 2), leaving room for the kernels that run concurrently with it -- the next frame's raycast / TSDF chain and, on
 * a multi-GPU rank, the NCCL all-gather of the block-list merge (4 there). Results do not depend on it. */
NVB_API int32_t nvb_mapper_set_esdf_reserved_sms(NvbMapper* m, int32_t reserved_sms);
NVB_API int32_t nvb_mapper_get_esdf_reserved_sms(const NvbMapper* m);

/* ---- Mesh (SURVEY.md section 8(f) rank 4: C/include/nvblox/mesh/mesh_integrator.h:39-162, C/src/mesh/mesh_integrator.cu,
 * C/src/mesh/mesh_integrator_appearance.cu). The mesh layer holds, per VoxelBlock that has triangles, vertices (3 floats),
 * flat per-vertex normals (3 floats), triangle indices into the block's vertices (triplets) and -- after a colour update --
 * one RGBA colour per vertex (MeshBlock, C/include/nvblox/mesh/mesh_block.h:32-83). A block's triangles come out in
 * x-major voxel order (the reference's order within a block is an atomicAdd race, marching_cubes_impl.cuh:11-29). */
typedef struct {
  float min_weight;          /* mesh_integrator_min_weight, 1e-4 (C/include/nvblox/mesh/mesh_integrator_params.h:22-24) */
  int32_t weld_vertices;     /* mesh_integrator_weld_vertices, true (mesh_integrator_params.h:25-27) */
  float cutoff_distance_vox; /* MeshIntegrator::cutoff_distance_vox_, 5 (mesh_integrator.h:129) */
} NvbMeshParams;
NVB_API void nvb_default_mesh_params(NvbMeshParams* p);
NVB_API int32_t nvb_mapper_set_mesh_params(NvbMapper* m, const NvbMeshParams* p);
NVB_API int32_t nvb_mapper_get_mesh_params(const NvbMapper* m, NvbMeshParams* p);
/* Mapper::updateColorMesh(UpdateFullLayer) (C/src/mapper/mapper.cpp:371-406): re-meshes the blocks touched since the last
 * call (or every block) and colours them from the colour layer; a no-op for an occupancy mapper. */
NVB_API int32_t nvb_mapper_update_mesh(NvbMapper* m, int32_t update_full_layer);
/* MeshIntegrator::integrateBlocksGPU (mesh_integrator.cu:66-108) on an explicit list of block indices (host, triples; the
 * ones missing from the TSDF layer are skipped), optionally followed by MeshIntegrator::updateAppearance on the same list. */
NVB_API int32_t nvb_mesh_integrate_blocks(NvbMapper* m, const int32_t* blocks_xyz_host, int32_t num_blocks, int32_t update_color);
/* MeshIntegrator::updateAppearance(colour layer, block list, mesh layer) (mesh_integrator_appearance.cu:71-96,281-380). */
NVB_API int32_t nvb_mesh_update_color(NvbMapper* m, const int32_t* blocks_xyz_host, int32_t num_blocks);
/* Sizes of the listed mesh blocks: sizes_out[3 i ..] = {vertices, triangle indices, colours}, or -1s if block i has no mesh
 * block. The block indices of the layer: nvb_layer_block_indices(m, NVB_LAYER_MESH, ...). A negative num_blocks is
 * NVB_ERR_INVALID_ARGUMENT. */
NVB_API int32_t nvb_mesh_block_sizes(NvbMapper* m, const int32_t* blocks_xyz_host, int32_t num_blocks, int32_t* sizes_out);
/* The listed mesh blocks packed back to back in list order into host buffers (any of them may be NULL): 3 floats per
 * vertex / normal, one int32 per triangle index (relative to the block's first vertex), 4 bytes RGBA per colour.
 * caps = capacities of the buffers in {vertices, triangle indices, colours}. A negative num_blocks is NVB_ERR_INVALID_ARGUMENT. */
NVB_API int32_t nvb_mesh_get_blocks(NvbMapper* m, const int32_t* blocks_xyz_host, int32_t num_blocks, float* vertices_out,
                                    float* normals_out, int32_t* triangles_out, uint8_t* colors_out, const int64_t caps[3]);
/* out = {arena capacity, fill level, vertices emitted by the last update, reserved} in vertices. */
NVB_API int32_t nvb_mesh_arena_stats(NvbMapper* m, int64_t out[4]);

/* Mapper::do_depth_preprocessing / depth_preprocessing_num_dilations (C/include/nvblox/mapper/mapper_params.h:33-42, defaults
 * off / 4; Mapper::preprocessDepthImageAsync, C/src/mapper/mapper.cpp:335-352): when enabled, nvb_mapper_integrate_depth*
 * integrates (and keeps as the last view) a copy of the depth image whose invalid regions were dilated. */
NVB_API int32_t nvb_mapper_set_depth_preprocessing(NvbMapper* m, int32_t enable, int32_t num_dilations);
NVB_API int32_t nvb_mapper_get_depth_preprocessing(const NvbMapper* m, int32_t* enable, int32_t* num_dilations);
/* DepthPreprocessor::dilateInvalidRegionsAsync (C/src/sensors/depth_preprocessing.cpp; C/include/nvblox/sensors/
 * depth_preprocessing.h): pixels with depth < invalid_depth_threshold (the class default is 1e-2) are invalid; the invalid
 * mask is dilated num_dilations times with a 3x3 structuring element (replicated border) and every masked pixel is written
 * as invalid_depth_value (default 0). Device pointers, rows*cols floats, out_dev must not alias depth_dev; enqueued on the
 * mapper's stream. */
NVB_API int32_t nvb_depth_dilate_invalid(NvbMapper* m, const float* depth_dev, float* out_dev, int32_t rows, int32_t cols,
                                         int32_t num_dilations, float invalid_depth_threshold, float invalid_depth_value);

/* Device-resident merge of the ranks' updated-block lists (multi-GPU; SURVEY.md section 8(e); the reference has no counterpart:
 * it is single-GPU and keeps `updated_blocks` in a host std::vector, C/include/nvblox/mapper/internal/impl/mapper_impl.h:40-60).
 * A SEGMENT is an int32 device array [count, x0, y0, z0, x1, ...] of capacity cap_entries (1 + 3 * cap_entries ints).
 *  - nvb_mapper_append_frame_blocks: appends the block list of the last integrated frame to a segment, enqueued on the mapper's
 *    stream (no host synchronisation; the caller zeroes segment[0] when a batch starts);
 *  - nvb_blocks_union_segments: sorted unique union (x fastest, then y, then z) of num_segments gathered segments laid out every
 *    segment_stride_ints ints -- AABB, bitset marking and ordered compaction all sized on the device -- written to
 *    out_xyz_dev / out_count_dev; enqueued on `stream` (a cudaStream_t; NULL = the mapper's stream), no host synchronisation;
 *  - nvb_blocks_union_status: synchronises and reports whether a union overflowed its bitset (1) -- a test / debug call. */
NVB_API int32_t nvb_mapper_append_frame_blocks(NvbMapper* m, int32_t* segment_dev, int32_t cap_entries);
NVB_API int32_t nvb_blocks_union_segments(NvbMapper* m, const int32_t* segments_dev, int32_t num_segments,
                                          int32_t segment_stride_ints, int32_t cap_entries, int32_t* out_xyz_dev,
                                          int32_t out_cap, int32_t* out_count_dev, void* stream);
NVB_API int32_t nvb_blocks_union_status(NvbMapper* m, int32_t* out_error);

/* Device-side join (no host synchronisation): work enqueued on nvb_mapper_stream() after this
 * call also waits for the ESDF wavefront, which runs on an internal side stream so that it
 * overlaps the next frame's TSDF chain. Needed before recording an event on the mapper's stream. */
NVB_API int32_t nvb_mapper_join_streams(NvbMapper* m);
/* The CUDA stream (cudaStream_t) all of the mapper's work is enqueued on
 * (Mapper's shared CudaStream, src/mapper/mapper.cpp:28-46). */
NVB_API void* nvb_mapper_stream(NvbMapper* m);

/* BlockLayer queries (C/include/nvblox/map/layer.h:76-311). All synchronising. */
NVB_API int32_t nvb_layer_num_blocks(NvbMapper* m, int32_t layer, int32_t* out_count);      /* numBlocks        */
NVB_API int32_t nvb_layer_block_indices(NvbMapper* m, int32_t layer, int32_t* out_xyz_host,
                                        int32_t cap, int32_t* out_count);                    /* getAllBlockIndices */
/* Storage of a layer's block slab: out = {capacity in blocks, high-water mark (slots handed out so far), free-stack size
 * (deallocated slots below the high-water mark, reused before fresh ones), hash-table size}. */
NVB_API int32_t nvb_layer_slab_stats(NvbMapper* m, int32_t layer, int64_t out[4]);
/* getBlockAtIndex(...)->voxels copied to host: out_host receives n blocks of
 * block_bytes (4096 TSDF / 10240 ESDF); found[i] = 0 for unallocated indices
 * (their output bytes are zero). block_bytes: 4096 TSDF / 10240 ESDF / 2048 occupancy. A negative n is
 * NVB_ERR_INVALID_ARGUMENT. */
NVB_API int32_t nvb_layer_get_blocks(NvbMapper* m, int32_t layer, const int32_t* xyz_host,
                                     int32_t n, void* out_host, uint8_t* found_host);
/* allocateBlockAtIndex + host->device copy of the voxels (tests, map loading). Each index carries its own block, so an
 * index listed twice is NVB_ERR_INVALID_ARGUMENT, as is a negative n; an index outside +-2^20 is NVB_ERR_INDEX_RANGE.
 * Either way nothing is written. */
NVB_API int32_t nvb_layer_set_blocks(NvbMapper* m, int32_t layer, const int32_t* xyz_host,
                                     int32_t n, const void* in_host);
/* getBlockAtIndex(index).get(): raw device pointer of a block, NULL if absent.
 * Valid until the layer's slab grows or the map is cleared. An ESDF block's bytes are the split form (cell plane, then
 * flag plane; see the top of this file), not voxels[8][8][8] of NvbEsdfVoxel: code that reads ESDF blocks on the device as
 * EsdfVoxel, like the dense grid of nvblox_ros's EsdfAndGradients service (voxelLayerToDenseVoxelGridInAABBAsync), uses
 * nvb_esdf_dense_grid_in_aabb instead. */
NVB_API int32_t nvb_layer_block_device_ptr(NvbMapper* m, int32_t layer, const int32_t xyz[3],
                                           void** out_ptr);
NVB_API int32_t nvb_layer_block_bytes(int32_t layer);

/* Map files: Mapper::saveLayerCake / Mapper::loadMap (src/mapper/mapper.cpp:636-687) in the reference's .nvblx format, an
 * SQLite database with the tables <layer>_metadata (rows 'type' and 'block_size') and <layer>_data (one row of index_x,
 * index_y, index_z and the block's voxels[8][8][8], byte for byte, per block) for tsdf_layer, esdf_layer, occupancy_layer,
 * freespace_layer, color_layer and feature_layer. SQLite is loaded from libsqlite3.so.0 on first use; without it both calls
 * fail with NVB_ERR_IO, which also stands for a file that cannot be opened, read or written (the reference logs and
 * returns false).
 *
 * Save joins the mapper's streams and truncates `path`. All six tables are written, one transaction per layer; a layer
 * this mapper does not hold (the other projective layer, freespace without NVB_PROJECTIVE_TSDF_WITH_FREESPACE, colour
 * before its first use, features always) is an empty table with the block size. Rows go in (x, y, z) block-index order,
 * so two saves of equal maps hold the same rows whatever the allocation history (the reference's order is its hash's). */
NVB_API int32_t nvb_mapper_save_map(NvbMapper* m, const char* path);
/* Load replaces the map with the file's: the projective layer this mapper holds (tsdf_layer or occupancy_layer), the
 * ESDF, colour (TSDF mappers) and freespace (NVB_PROJECTIVE_TSDF_WITH_FREESPACE). Other tables, feature_layer always,
 * are skipped, and the call still succeeds: loaded_blocks (optional, by NvbLayer id 0-4, then [5] the feature layer)
 * reports the blocks loaded per layer, 0 for a skipped table. The voxel size becomes the file's block_size / 8; when it
 * changes, the cached viewpoint of the projective integrator is dropped. Every consumer's next update covers every block
 * (a fresh BlocksToUpdateTracker); a TSDF mapper ends with a full colour-mesh update. The freespace integrator's last
 * update time, the last integrated view and the cleared-block set are kept. The file is validated before the map is
 * touched, and a failed load leaves the map as it was:
 *  - NVB_ERR_IO: no file, not a map file, no tsdf_layer table, a layer without block_size, block sizes that differ, a
 *    blob of other than nvb_layer_block_bytes(layer) bytes, or an index twice;
 *  - NVB_ERR_INDEX_RANGE: an index outside +-2^20;
 *  - NVB_ERR_CAPACITY: a layer beyond 2^28 blocks. */
NVB_API int32_t nvb_mapper_load_map(NvbMapper* m, const char* path, int32_t loaded_blocks[6]);
/* io::outputVoxelLayerToPly's points (io/pointcloud_io.cpp:23-73) of NVB_LAYER_TSDF (weight > 1e-4, intensity distance),
 * NVB_LAYER_OCCUPANCY (p = probabilityFromLogOdds(log_odds) > 0.5, intensity p), NVB_LAYER_FREESPACE (every voxel,
 * intensity is_high_confidence_freespace) or NVB_LAYER_ESDF (observed, intensity voxel_size * sqrt(squared_distance_vox),
 * negative inside): 4 floats {x, y, z, intensity} per point at the voxel centre, into xyzi (host or device memory). The
 * order is canonical: blocks in (x, y, z) block-index order, then voxels in x, y, z order (the reference follows its
 * hash). *n = the number of points; with cap < *n nothing is written. */
NVB_API int32_t nvb_layer_export_points(NvbMapper* m, int32_t layer, int32_t memory, float* xyzi, int64_t cap, int64_t* n);

/* ---- Point queries: the map read at arbitrary points on the GPU. A query reads the map and never writes it.
 * Points are n x 3 floats (x, y, z); spheres n x 4 floats (x, y, z, radius). A point's voxel is the one
 * getBlockAndVoxelIndexFromPositionInLayer names (C/include/nvblox/core/internal/impl/indexing_impl.h:37-49).
 * Deviations from the reference, whose behaviour on these inputs is undefined or accidental:
 *  - a point with a non-finite coordinate, or whose block index lies outside the hash's +-2^20 key range, is a miss;
 *  - the mappers of one nvb_query_* call must be on the same device (NVB_ERR_INVALID_ARGUMENT otherwise).
 * Ordering: a query runs after all work already enqueued on every mapper it reads (including a pending ESDF update), and
 * each of those mappers' later work runs after the query. With device buffers nothing synchronises the host: the waits are
 * event hops. n == 0 launches nothing; a bad layer or a null pointer is NVB_ERR_INVALID_ARGUMENT. */
/* VoxelBlockLayer::getVoxels / getVoxelsGPU (C/include/nvblox/map/layer.h:265-295, map/internal/cuda/impl/layer_impl.cuh:29-80)
 * on any voxel layer (TSDF, ESDF, occupancy, freespace, colour): out_voxels receives n voxels as stored (NvbTsdfVoxel,
 * NvbEsdfVoxel, float log-odds, NvbFreespaceVoxel, NvbColorVoxel), written only where out_success[i] = 1. All three buffers
 * are in `memory`; host buffers are written when the call returns, device ones are enqueued on the mapper's stream. */
NVB_API int32_t nvb_layer_query_voxels(NvbMapper* m, int32_t layer, const float* xyz, int32_t memory, int64_t n,
                                       void* out_voxels, uint8_t* out_success);
/* interpolation::interpolateOnCPU (C/src/interpolation/interpolation_3d.cpp) of the TSDF, ESDF or occupancy layer, on the GPU:
 * trilinear interpolation of the 8 voxels around each point (the low corner is the voxel of p - voxel_size / 2; they may lie
 * in up to 8 blocks). TSDF: `distance`, every voxel needs weight > 1e-4. ESDF: sqrt(squared_distance_vox) -- unsigned and in
 * voxels, as in the reference --, every voxel needs `observed`. Occupancy: the probability exp(l) / (1 + exp(l)). A point
 * fails (out_success 0, value 0) when a block is missing or a voxel is invalid. The weighted sum q . (T . m) runs left to
 * right over the non-zero entries of the reference's 8x8 table. Buffers in `memory`, as nvb_layer_query_voxels. */
NVB_API int32_t nvb_layer_interpolate(NvbMapper* m, int32_t layer, const float* xyz, int32_t memory, int64_t n,
                                      float* out_values, uint8_t* out_success);
/* nvblox_torch's ESDF sphere query (nvblox_torch/cpp/src/sdf_query.cu:63-205) over the ESDF layers of num_mappers mappers
 * (at most 16). Device buffers. out is n x 4 {gx, gy, gz, d} with_gradient, else n x 1 {d}. Per mapper holding the sphere's
 * voxel: unobserved -> d = 100; else distance = +-voxel_size * sqrt(squared_distance_vox) (negative inside), d = distance -
 * radius, gradient = (-voxel_size / distance) * parent_direction, or 0 when distance <= 1e-6. With several mappers the
 * minimum is kept from 100 down: a mapper whose d exceeds the running minimum writes that minimum and leaves the gradient.
 * Outputs a sphere never writes keep their contents (the caller pre-fills them, nvblox_torch uses 100). The query is
 * enqueued on caller_stream (a cudaStream_t; NULL is the default stream, as in CUDA): it also runs after the work already
 * there, and that stream's next work follows it. One mapper takes the single-mapper rules (no minimum). */
NVB_API int32_t nvb_query_esdf(NvbMapper* const* mappers, int32_t num_mappers, const float* spheres_xyzr, int64_t n,
                               int32_t with_gradient, float* out, void* caller_stream);
/* nvblox_torch's TSDF point query (sdf_query.cu:240-318): out n x 2 {distance, weight}. One mapper: written where the voxel
 * exists. Several: the smallest distance and the weight at it, starting from {100, 0}. Ordering as nvb_query_esdf. */
NVB_API int32_t nvb_query_tsdf(NvbMapper* const* mappers, int32_t num_mappers, const float* xyz, int64_t n, float* out,
                               void* caller_stream);
/* nvblox_torch's occupancy point query (sdf_query.cu:320-351) over the mappers' occupancy layers: out n x 1, the largest
 * log-odds of the voxels that exist, starting from logOddsFromProbability(0). Ordering as nvb_query_esdf. */
NVB_API int32_t nvb_query_occupancy(NvbMapper* const* mappers, int32_t num_mappers, const float* xyz, int64_t n, float* out,
                                    void* caller_stream);

/* Counters of the last ESDF update (for the roofline's algorithmic bytes):
 * [0] blocks marked, [1] blocks with sites, [2] blocks to clear, [3] clear-pass
 * candidate blocks, [4] blocks cleared, [5] swept blocks, [6] (block,direction)
 * face passes, [7] rings. Synchronising. */
NVB_API int32_t nvb_mapper_last_esdf_stats(NvbMapper* m, int64_t out[8]);

/* Time split of the last ESDF wavefront launch as seen by CTA 0 (ns): [0] grid barriers,
 * [1] face-propagation phases, [2] scan + sweep phases, [3] number of grid barriers. Synchronising. */
NVB_API int32_t nvb_mapper_esdf_time_split(NvbMapper* m, int64_t out[4]);

/* Blocks the clear pass of the last ESDF update actually read (clearAllInvalidKernel's candidates,
 * nvblox/src/integrators/esdf_integrator.cu:1587-1647, minus those whose parent box holds no to-clear block; the
 * `clear_candidates` statistic keeps counting the reference's candidates). */
NVB_API int32_t nvb_mapper_esdf_clear_blocks_read(NvbMapper* m, int64_t* out);

/* The exchange-slab wavefront's own-block fetches in the last ESDF update: [0] candidates whose block was fetched split
 * (boundary planes first), [1] of those, the ones that changed and fetched the rest of their block. Synchronising. */
NVB_API int32_t nvb_mapper_esdf_split_stats(NvbMapper* m, int64_t out[2]);

/* Debug: work time (ns) of the slowest CTA in each barrier-delimited phase of the last wavefront. */
NVB_API int32_t nvb_mapper_debug_phase_max(NvbMapper* m, int64_t* out, int32_t cap);

/* Per-stage device time of the frames since the last reset, measured with CUDA
 * events on the mapper's stream when profiling is enabled (same names as the
 * reference's timers: "tsdf/integrate", "esdf/integrate", ...;
 * projective_integrator_impl.cuh:230-270, esdf_integrator.cu:224-252).
 * stage ids: 0 view raycast, 1 block compaction+allocation, 2 tsdf update,
 * 3 esdf allocate+mark, 4 esdf clear, 5 esdf compute. out_ms / out_calls have 6 entries. */
NVB_API int32_t nvb_mapper_enable_profiling(NvbMapper* m, int32_t enable);
NVB_API int32_t nvb_mapper_stage_times(NvbMapper* m, double* out_ms, int64_t* out_calls,
                                       int32_t reset);
/* Number of kernels this library launched on behalf of the mapper since creation. */
NVB_API int64_t nvb_mapper_kernel_launches(const NvbMapper* m);

#ifdef __cplusplus
}
#endif
#endif /* NVBLOX_B200_H_ */
