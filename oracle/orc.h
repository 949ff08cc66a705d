/*
 * oracle/orc.h -- CPU ORACLE for the MaskFusion per-frame dense pipeline.
 *
 * THIS IS TEST INFRASTRUCTURE, NOT THE PRODUCT.  Only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
 * may load this library.  The product (maskfusion_b200/) never links, imports
 * or executes anything in oracle/.
 *
 * It is a plain-C restatement (IEEE fp32, no FMA contraction, fixed operation
 * order) of the reference's CUDA kernels (Core/Cuda/ *.cu), GLSL passes
 * (Core/Shaders/) and the host maths that drives them (Core/Utils/
 * RGBDOdometry.cpp, Core/Model/Model.cpp, Core/MaskFusion.cpp).  Every function
 * cites the reference file:line it follows.
 *
 * PARITY PINNING: the reference ships no tests, golden vectors or fixtures
 * (SURVEY.md section 4).  The CUDA half of the oracle (maps, pyramids, ICP / RGB /
 * SO3 reductions, edge-ness) is pinned against the reference's own kernels
 * recompiled for sm_90a (oracle/_ref, built by oracle/Makefile.ref) on the GPU
 * box; the GLSL half cannot be executed anywhere in this environment (no
 * OpenGL) => "parity unpinned" for those passes; their semantics are fixed in
 * writing in DESIGN.md (rules N1..N14 of SURVEY.md Appendix A).
 *
 * Conventions
 *   images: row-major, index y*W + x.
 *   planar maps (reference DeviceArray2D<float> 3*rows x cols): plane p at
 *       [(p*rows + y)*cols + x]                     (cudafuncs.cu:124-126)
 *   "tex4" images: interleaved RGBA32F, [ (y*W + x)*4 + c ]   (GL textures)
 *   surfels: 12 floats each: pos.xyz conf | color unused initTime lastTime |
 *       normal.xyz radius                           (Model.h:190-192)
 *   poses: float[16] ROW-major 4x4 (T[r*4+c]).
 */
#ifndef ORC_H
#define ORC_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct { float fx, fy, cx, cy; } orc_cam;

/* ---- deterministic transcendental definitions (shared semantics with the
 *      CUDA build, which restates the same polynomials) ---- */
float orc_expf(float x);
float orc_acosf(float x);

/* ---- small host maths ---- */
void orc_pose_inverse(const float* T, float* Tinv);             /* rigid inverse */
void orc_pose_mul(const float* A, const float* B, float* C);
orc_cam orc_cam_level(orc_cam c, int level);                    /* types.cuh:94-98 */

/* ================= maps & pyramids (Core/Cuda/cudafuncs.cu) ============== */
void orc_bilateral(const float* depth, float* out, int W, int H);            /* depth_bilateral_metric.frag:30-76 */
void orc_pyrdown_gauss_f(const float* src, int sw, int sh, float* dst);      /* cudafuncs.cu:333-364 */
void orc_pyrdown_gauss_u8(const uint8_t* src, int sw, int sh, uint8_t* dst); /* cudafuncs.cu:534-564 */
void orc_vmap(const float* depth, int W, int H, orc_cam cam, float cutoff, float* vmap /*3*H*W*/);   /* :109-134 */
void orc_nmap(const float* vmap, int W, int H, float* nmap);                                           /* :152-189 */
void orc_copy_maps(const float* vtex4, const float* ntex4, int W, int H, float* vmap, float* nmap);   /* :271-311 */
void orc_resize_map(const float* in, int sw, int sh, int normalize, float* out);                       /* :366-417 */
void orc_transform_maps(float* vmap, float* nmap, int W, int H, const float* R9, const float* t3);    /* :207-249 */
void orc_vertices_to_depth(const float* vtex4, int W, int H, float cutoff, float* depth);             /* :602-613 */
void orc_rgb_to_intensity(const uint8_t* rgb3, int W, int H, uint8_t* out);                           /* :626-639 */
void orc_sobel(const uint8_t* src, int W, int H, int16_t* dx, int16_t* dy);                           /* :658-683 */
void orc_project_points(const float* depth, int W, int H, orc_cam cam, float* cloud3);                /* :718-736 */

/* ================= reductions (Core/Cuda/reduce.cu) ====================== */
/* out29: 27 upper-triangular products (row-major i<=j<7), residual, inliers */
void orc_icp_step(const float* Rcurr9, const float* tcurr3,
                  const float* vmap_curr, const float* nmap_curr,
                  const float* Rprev_inv9, const float* tprev3, orc_cam cam,
                  const float* vmap_g_prev, const float* nmap_g_prev,
                  float distThres, float angleThres, int W, int H, double* out29);     /* reduce.cu:259-444 */
typedef struct { int16_t zx, zy, ox, oy; float diff; int32_t valid; } orc_dataterm;    /* types.cuh:75-81 */
void orc_rgb_residual(float minScale, const int16_t* dIdx, const int16_t* dIdy,
                      const float* lastDepth, const float* nextDepth,
                      const uint8_t* lastImage, const uint8_t* nextImage,
                      orc_dataterm* corres, float maxDepthDelta, const float* kt3,
                      const float* krkinv9, int W, int H, int* count, int* sigmaSum);  /* reduce.cu:774-997 */
void orc_rgb_step(const orc_dataterm* corres, float sigma, const float* cloud3,
                  float fx, float fy, const int16_t* dIdx, const int16_t* dIdy,
                  float sobelScale, int W, int H, double* out29);                      /* reduce.cu:529-713 */
void orc_so3_step(const uint8_t* lastImage, const uint8_t* nextImage,
                  const float* imageBasis9, const float* kinv9, const float* krlr9,
                  int W, int H, double* out11);                                        /* reduce.cu:999-1202 */

/* ================= odometry driver (Core/Utils/RGBDOdometry.cpp) ========= */
typedef struct orc_odom orc_odom;   /* per-model RGBDOdometry state */
typedef struct {
    int rgbOnly; float icpWeight; int pyramid; int fastOdom; int so3;
} orc_track_params;

/* ================= surfel passes (Core/Shaders, Core/Model) ============== */
/* index map: index_map.vert/.frag, ModelProjection.cpp:100-152 */
void orc_predict_indices(const float* surfels, int count, const float* pose, orc_cam cam,
                         int W, int H, float maxDepth, int time, int timeDelta,
                         uint32_t* idx, float* vertConf4, float* colorTime4, float* normRad4);
/* data association: data.vert/.geom/.frag, Model.cpp:466-581.
 * updateId[p]  (x-major pixel order p = x*H + y): 0 ignore, 1 merge, 2 new.
 * best[p] = surfel id merged into; meas[p*12..] = the emitted vertex. */
void orc_data_associate(const uint8_t* rgb3, const float* depthRaw, const float* depthFilt,
                        const uint8_t* mask, const uint32_t* idx, const float* vertConf4,
                        const float* normRad4, const float* pose, orc_cam cam, int W, int H,
                        float maxDepth, int time, float weighting, uint8_t maskID,
                        uint8_t* updateId, uint32_t* best, float* meas);
/* update.vert with N4 collision rule (first pixel in x-major order wins) */
void orc_fuse_update(float* surfels, int count, const uint8_t* updateId, const uint32_t* best,
                     const float* meas, int W, int H, int time);
/* copy_unstable.vert/.geom, Model.cpp:649-772.  Returns new count; out holds
 * survivors (old order) then new-unstable vertices (x-major pixel order). */
int orc_clean(const float* surfels, int count, const uint8_t* updateId, const float* meas,
              const uint32_t* idx, const float* vertConf4, const float* colorTime4,
              const float* depthFilt, const uint8_t* mask, const float* pose, orc_cam cam,
              int W, int H, int time, int timeDelta, float confThreshold, float outlierCoeff,
              uint8_t maskID, float* out, int capacity);
/* splat.vert + combo_splat.frag, ModelProjection.cpp:187-268 */
void orc_combined_predict(const float* surfels, int count, const float* pose, orc_cam cam,
                          int W, int H, float maxDepth, float confThreshold, int time, int maxTime,
                          int timeDelta, uint8_t* image4, float* vertexConf4, float* normalRad4,
                          uint16_t* timeTex);
/* fill_{vertex,normal,rgb}.frag, FillIn.cpp:43-166 */
void orc_fill_in(const float* vertexConf4, const float* normalRad4, const uint8_t* image4,
                 const float* depthFilt, const uint8_t* rgb3, orc_cam cam, int W, int H,
                 int passthroughVN, int passthroughImg,
                 float* fillVertex4, float* fillNormal4, uint8_t* fillImage4);
/* resize.frag + MaskFusion.cpp:630-648 */
int orc_requires_fill_in(const uint8_t* image4, int W, int H, float ratio);
/* vertex_feedback.vert/.geom + init_unstable.vert, Model.cpp:240-285 */
int orc_init_model(const uint8_t* rgb3, const float* depthRaw, const float* depthFilt,
                   orc_cam cam, int W, int H, int time, float maxDepth, float* out, int capacity);
/* splat_models.vert + combo_splat_models.frag, GlobalProjection.cpp:43-107.
 * keys: per pixel packed (fragDepth bits << 32 | draw order), caller keeps. */
void orc_global_projection_begin(int W, int H, uint64_t* keys);
void orc_global_projection_add(const float* surfels, int count, const float* pose, orc_cam cam,
                               int W, int H, float maxDepth, float confThreshold, int time,
                               int maxTime, int timeDelta, uint32_t drawBase, uint64_t* keys);

/* ================= geometric segmentation (Core/Cuda/segmentation.cu) ==== */
void orc_geometric_edges(const float* vmap, const float* nmap, int W, int H, float wD, float wC, float* out); /* :122-177 */
void orc_threshold(const float* in, int n, float thr, uint8_t* out);                                          /* :257-262 */
void orc_invert(const uint8_t* in, int n, uint8_t* out);                                                      /* :264-269 */
void orc_morph_close(uint8_t* data, uint8_t* buf, int W, int H, int radius, int iterations);                  /* :217-255,334-354 */

#ifdef __cplusplus
}
#endif
#endif
