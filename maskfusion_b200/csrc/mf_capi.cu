// mf_capi.cu -- the C ABI declared in include/maskfusion_b200.h (drop-in boundary).
// Every entry point that can fail runs inside MF_TRY / MF_CATCH (mf_kernels.h), which turns C++ exceptions and CUDA
// errors into a non-zero return + mf_last_error(); poses cross the boundary in Eigen's column-major layout.
#include "mf_host.h"
#include <string.h>
#include <stdio.h>
#include <zlib.h>
#include <limits.h>
#include <new>
#include <stack>

using namespace mfb;
namespace mfb { bool decodeJPEG(const uint8_t* data, size_t size, int& W, int& H, std::vector<uint8_t>& rgb, std::string& err); }   // mf_jpeg.cu

struct mf_context { std::unique_ptr<MaskFusion> mf; };

// one message per calling thread: contexts and Mask R-CNN handles driven from different threads never see each other's errors
static thread_local std::string g_err;
void mf_set_error(const std::string& msg) { g_err = msg; }
extern "C" const char* mf_last_error(void) { return g_err.c_str(); }
extern "C" const char* mf_cnn_last_error(void) { return g_err.c_str(); }       // the same message, under the name older bindings read
extern "C" int mf_abi_version(void) { return MF_ABI_VERSION; }

// every entry point first picks up a tracked pose that is still in flight (-static frames return before it has arrived); inside MF_TRY
static void mf_finalise(mf_context* ctx)
{
    // the calling thread may have another device current (several contexts per process): every entry point selects its own
    cudaCheck(cudaSetDevice(ctx->mf->device), "cudaSetDevice");
    ctx->mf->finalisePending();
}
#define MF_NEED(ctx) if (!(ctx) || !(ctx)->mf) { mf_set_error("null context"); return -1; } mf_finalise(ctx);
#define MF_MODEL(ctx, i) if ((i) < 0 || (i) >= (int)(ctx)->mf->models.size()) { mf_set_error("model index out of range"); return -2; } Model* m = (ctx)->mf->models[i].get();

#define MF_OWNED(m) if (!(m)->owned) { mf_set_error("model is owned by another rank (sharded mode): no device buffers here"); return -4; }
// the stage-wise calls work on the frame processed last, which frames still in the queue would no longer follow
#define MF_UNQUEUED(ctx, who)                                                                                                                  \
    if ((ctx)->mf->queued) {                                                                                                                   \
        mf_set_error(std::string(who) + ": " + std::to_string((ctx)->mf->queued) + " frame(s) are queued (mf_set_frame_queue); the stage-wise calls " \
                "run on a context with no frames queued");                                                                                      \
        return -6;                                                                                                                             \
    }

static Mat4 fromColMajor(const float* p) { Mat4 r; for (int rr = 0; rr < 4; ++rr) for (int c = 0; c < 4; ++c) r.m[rr * 4 + c] = p[c * 4 + rr]; return r; }
static void toColMajor(const Mat4& T, float* p) { for (int rr = 0; rr < 4; ++rr) for (int c = 0; c < 4; ++c) p[c * 4 + rr] = T.m[rr * 4 + c]; }

extern "C" void mf_config_defaults(mf_config* c, int width, int height)
{
    memset(c, 0, sizeof *c);
    c->width = width; c->height = height;
    if (width == 640 && height == 480) { c->fx = 528; c->fy = 528; c->cx = 320; c->cy = 240; }        // MainController.cpp:124-125
    else { c->fx = 528.f * width / 640.f; c->fy = c->fx; c->cx = width / 2.f; c->cy = height / 2.f; }
    c->depthCutoff = 4.0f; c->maxDepthProcessed = 20.0f; c->icpWeight = 20.0f;
    c->rgbOnly = 0; c->pyramid = 1; c->fastOdom = 0; c->so3 = 1; c->frameToFrameRGB = 0;
    c->confGlobal = 10.0f; c->confObject = 0.01f;
    c->timeDelta = INT_MAX / 2;
    c->outlierCoeff = 0.1f;
    c->capacityGlobal = 3072 * 3072; c->capacityObject = 1024 * 1024;
    c->enableMultipleModels = 0; c->trackAllModels = 0; c->modelSpawnOffset = 22;
    c->minRelSizeNew = 0.015f; c->maxRelSizeNew = 0.4f;
    c->segThreshold = 0.3f; c->segWeightDistance = 150.f; c->segWeightConvexity = 2.8f;
    c->segMorphEdgeIterations = 0; c->segMorphEdgeRadius = 1; c->segMorphMaskIterations = 0; c->segMorphMaskRadius = 2;
}

extern "C" mf_context* mf_create(const mf_config* cfg, int device, void* stream)
{
    MF_TRY
    if (!cfg) { mf_set_error("null config"); return nullptr; }
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) { mf_set_error(std::string("no CUDA device: this library has no CPU fallback (") + cudaGetErrorString(e) + ")"); return nullptr; }
    std::unique_ptr<MaskFusion> mf(new MaskFusion(*cfg, device, (cudaStream_t)stream));
    return new mf_context{std::move(mf)};
    MF_CATCH(nullptr)
}
extern "C" void mf_destroy(mf_context* ctx) { delete ctx; }

extern "C" int mf_process_frame(mf_context* ctx, const uint8_t* rgb, const float* depth, int64_t ts, const uint8_t* mask, const float* in_pose,
                                float weight_multiplier, int bootstrap)
{
    MF_TRY MF_NEED(ctx)
    if (!rgb || !depth || ts < 0) { mf_set_error("processFrame: rgb/depth must be non-null and timestamp >= 0 (MaskFusion.cpp:201-203)"); return -3; }
    Mat4 ip; if (in_pose) ip = fromColMajor(in_pose);
    ctx->mf->processFrame(rgb, depth, ts, mask, in_pose ? &ip : nullptr, weight_multiplier, bootstrap != 0, false);
    return 0;
    MF_CATCH(-1)
}
extern "C" int mf_process_frame_device(mf_context* ctx, const void* d_rgb, const void* d_depth, int64_t ts, const void* d_mask, const float* in_pose,
                                       float weight_multiplier, int bootstrap)
{
    MF_TRY MF_NEED(ctx)
    if (!d_rgb || !d_depth || ts < 0) { mf_set_error("processFrame: rgb/depth must be non-null and timestamp >= 0"); return -3; }
    Mat4 ip; if (in_pose) ip = fromColMajor(in_pose);
    ctx->mf->processFrame((const uint8_t*)d_rgb, (const float*)d_depth, ts, (const uint8_t*)d_mask, in_pose ? &ip : nullptr, weight_multiplier,
                          bootstrap != 0, true);
    return 0;
    MF_CATCH(-1)
}
extern "C" int mf_set_input_event(mf_context* ctx, void* ev)
{
    MF_TRY if (!ctx || !ctx->mf) { mf_set_error("null context"); return -1; } ctx->mf->inputReady = (cudaEvent_t)ev; return 0; MF_CATCH(-1)
}
extern "C" int mf_sync(mf_context* ctx) { MF_TRY MF_NEED(ctx) ctx->mf->sync(); return 0; MF_CATCH(-1) }
extern "C" int mf_tick(mf_context* ctx) { if (!ctx || !ctx->mf) return -1; return ctx->mf->tick; }
extern "C" int mf_set_frame_queue(mf_context* ctx, int length) { MF_TRY MF_NEED(ctx) ctx->mf->setFrameQueue(length); return 0; MF_CATCH(-1) }
extern "C" int mf_frame_queue_size(mf_context* ctx) { MF_TRY if (!ctx || !ctx->mf) { mf_set_error("null context"); return -1; } return ctx->mf->queued; MF_CATCH(-1) }
extern "C" int64_t mf_kernel_launches(mf_context* ctx) { if (!ctx || !ctx->mf) return -1; return ctx->mf->rec.launches; }

extern "C" int mf_model_count(mf_context* ctx) { if (!ctx || !ctx->mf) return -1; return (int)ctx->mf->models.size(); }
extern "C" int mf_model_id(mf_context* ctx, int i) { MF_TRY MF_NEED(ctx) MF_MODEL(ctx, i) return m->id; MF_CATCH(-1) }
extern "C" int mf_get_pose(mf_context* ctx, int i, float* p) { MF_TRY MF_NEED(ctx) MF_MODEL(ctx, i) toColMajor(m->pose, p); return 0; MF_CATCH(-1) }
extern "C" int mf_set_pose(mf_context* ctx, int i, const float* p) { MF_TRY MF_NEED(ctx) MF_MODEL(ctx, i) m->overridePose(fromColMajor(p)); return 0; MF_CATCH(-1) }
extern "C" int mf_model_set_conf_threshold(mf_context* ctx, int i, float t) { MF_TRY MF_NEED(ctx) MF_MODEL(ctx, i) m->confidenceThreshold = t; return 0; MF_CATCH(-1) }
extern "C" int mf_model_surfel_count(mf_context* ctx, int i) { MF_TRY MF_NEED(ctx) MF_MODEL(ctx, i) return (int)m->lastCount(); MF_CATCH(-1) }

extern "C" int mf_download_surfels(mf_context* ctx, int i, float* out, int max_surfels)
{
    MF_TRY MF_NEED(ctx) MF_MODEL(ctx, i) MF_OWNED(m)
    MaskFusion* o = ctx->mf.get();
    uint32_t n = m->lastCount();
    if ((int)n > max_surfels) n = (uint32_t)max_surfels;
    if (!n) return 0;
    DevBuf<float4> tmp; tmp.alloc((size_t)n * 3);
    launch_planes_to_aos(m->current(), n, tmp, o->on());
    cudaCheck(cudaMemcpyAsync(out, tmp.p, (size_t)n * 48, cudaMemcpyDeviceToHost, o->stream), "surfel D2H");
    o->sync();
    return (int)n;
    MF_CATCH(-1)
}
extern "C" int mf_upload_surfels(mf_context* ctx, int i, const float* in, int n)
{
    MF_TRY MF_NEED(ctx) MF_MODEL(ctx, i) MF_OWNED(m)
    MaskFusion* o = ctx->mf.get();
    if (n < 0 || (uint32_t)n > m->capacity) { mf_set_error("upload exceeds model capacity"); return -4; }
    if (n) {
        DevBuf<float4> tmp; tmp.alloc((size_t)n * 3);
        cudaCheck(cudaMemcpyAsync(tmp.p, in, (size_t)n * 48, cudaMemcpyHostToDevice, o->stream), "surfel H2D");
        launch_aos_to_planes(tmp, (uint32_t)n, m->current(), o->on());
        o->sync();
    }
    uint32_t c = (uint32_t)n;
    cudaCheck(cudaMemcpyAsync(m->dCount(), &c, sizeof c, cudaMemcpyHostToDevice, o->stream), "count H2D");
    o->sync();
    return 0;
    MF_CATCH(-1)
}
extern "C" int mf_pose_log_size(mf_context* ctx, int i) { MF_TRY MF_NEED(ctx) MF_MODEL(ctx, i) return (int)(m->poseLog.size() / 8); MF_CATCH(-1) }
extern "C" int mf_get_pose_log(mf_context* ctx, int i, double* out8, int max_entries)
{
    MF_TRY MF_NEED(ctx) MF_MODEL(ctx, i)
    int n = (int)(m->poseLog.size() / 8); if (n > max_entries) n = max_entries;
    memcpy(out8, m->poseLog.data(), (size_t)n * 8 * sizeof(double));
    return n;
    MF_CATCH(-1)
}

// MaskFusion::exportPoses (MaskFusion.cpp:849-881): "<dir>poses-<id>.txt", one line per frame: seconds x y z qx qy qz qw, fixed, 6 decimals
extern "C" int mf_export_poses(mf_context* ctx, const char* export_dir)
{
    MF_TRY MF_NEED(ctx)
    if (!export_dir) { mf_set_error("export_poses: null directory"); return -2; }
    ctx->mf->sync();
    int written = 0;
    // active models, then the inactivated ones the keep rule retained (MaskFusion.cpp:849-881 walks models and inactiveModels)
    std::vector<Model*> all;
    for (auto& m : ctx->mf->models) all.push_back(m.get());
    for (auto& m : ctx->mf->inactiveModels) all.push_back(m.get());
    for (Model* m : all) {
        const std::string filename = std::string(export_dir) + "poses-" + std::to_string((int)m->id) + ".txt";
        FILE* fp = fopen(filename.c_str(), "w");
        if (!fp) { mf_set_error("cannot write " + filename); return -3; }
        for (size_t e = 0; e + 8 <= m->poseLog.size(); e += 8) {
            fprintf(fp, "%.6f", m->poseLog[e] * 1e-6);
            for (int k = 1; k < 8; ++k) fprintf(fp, " %.6f", (double)(float)m->poseLog[e + k]);      // the log holds Eigen floats (Model.h pose log)
            fprintf(fp, "\n");
        }
        fclose(fp);
        ++written;
    }
    return written;
    MF_CATCH(-1)
}

// ---- per-stage entry points ----
extern "C" int mf_set_frame(mf_context* ctx, const uint8_t* rgb, const float* depth, const uint8_t* mask)
{
    MF_TRY MF_NEED(ctx) MF_UNQUEUED(ctx, "set_frame")
    MaskFusion* o = ctx->mf.get();
    if (!mask) o->mask.zero(o->stream);
    o->setFrame(rgb, depth, mask, false);
    o->generateCUDATextures();
    return 0;
    MF_CATCH(-1)
}
extern "C" int mf_model_perform_tracking(mf_context* ctx, int i, float* transform16)
{
    MF_TRY MF_NEED(ctx) MF_MODEL(ctx, i) MF_OWNED(m) MF_UNQUEUED(ctx, "perform_tracking")
    std::vector<Model*> ms{m};
    ctx->mf->trackModels(ms);
    ctx->mf->finalisePending();
    if (transform16) toColMajor(m->lastTransform, transform16);
    return 0;
    MF_CATCH(-1)
}
extern "C" int mf_model_predict_indices(mf_context* ctx, int i, int time)
{
    MF_TRY MF_NEED(ctx) MF_MODEL(ctx, i) MF_OWNED(m) MF_UNQUEUED(ctx, "predict_indices")
    m->predictIndices(time, ctx->mf->cfg.maxDepthProcessed, ctx->mf->cfg.timeDelta); return 0;
    MF_CATCH(-1)
}
extern "C" int mf_model_fuse(mf_context* ctx, int i, int time, float depth_cutoff, float weight_multiplier)
{
    MF_TRY MF_NEED(ctx) MF_MODEL(ctx, i) MF_OWNED(m) MF_UNQUEUED(ctx, "fuse")
    m->fuse(time, depth_cutoff, weight_multiplier); return 0;
    MF_CATCH(-1)
}
extern "C" int mf_model_clean(mf_context* ctx, int i, int time)
{
    MF_TRY MF_NEED(ctx) MF_MODEL(ctx, i) MF_OWNED(m) MF_UNQUEUED(ctx, "clean")
    m->clean(time, ctx->mf->cfg.timeDelta, ctx->mf->cfg.maxDepthProcessed); return 0;
    MF_CATCH(-1)
}
extern "C" int mf_model_combined_predict(mf_context* ctx, int i, int time, int max_time)
{
    MF_TRY MF_NEED(ctx) MF_MODEL(ctx, i) MF_OWNED(m) MF_UNQUEUED(ctx, "combined_predict")
    m->combinedPredict(ctx->mf->cfg.maxDepthProcessed, time, max_time, ctx->mf->cfg.timeDelta); return 0;
    MF_CATCH(-1)
}
extern "C" int mf_model_init_from_frame(mf_context* ctx, int i, int time)
{
    MF_TRY MF_NEED(ctx) MF_MODEL(ctx, i) MF_OWNED(m) MF_UNQUEUED(ctx, "init_from_frame")
    m->initialise(time); return 0;
    MF_CATCH(-1)
}

// ---- read-back ----
template <typename T>
static void d2h(MaskFusion* o, void* dst, const T* src, size_t n)
{
    if (!dst) return;
    cudaCheck(cudaMemcpyAsync(dst, src, n * sizeof(T), cudaMemcpyDeviceToHost, o->stream), "D2H");
}
static void planarOut(MaskFusion* o, const float4* map, int P, float* out)
{
    if (!out) return;
    launch_map_to_planar(map, P, o->scratch, o->on());
    cudaCheck(cudaMemcpyAsync(out, o->scratch.p, (size_t)P * 3 * sizeof(float), cudaMemcpyDeviceToHost, o->stream), "D2H");
    o->sync();
}
extern "C" int mf_download_filtered_depth(mf_context* ctx, float* out)
{
    MF_TRY MF_NEED(ctx) d2h(ctx->mf.get(), out, ctx->mf->depthFilt, ctx->mf->P); ctx->mf->sync(); return 0; MF_CATCH(-1)
}
extern "C" int mf_download_frame_maps(mf_context* ctx, int level, float* depth, float* vmap, float* nmap)
{
    MF_TRY MF_NEED(ctx)
    MaskFusion* o = ctx->mf.get();
    if (level < 0 || level > 2) { mf_set_error("level out of range"); return -2; }
    int Pl = (o->W >> level) * (o->H >> level);
    d2h(o, depth, level == 0 ? o->depthFilt : o->depthPyr[level].p, Pl); o->sync();
    planarOut(o, o->vmap[level], Pl, vmap);
    planarOut(o, o->nmap[level], Pl, nmap);
    return 0;
    MF_CATCH(-1)
}
extern "C" int mf_download_model_maps(mf_context* ctx, int i, int level, float* vmap, float* nmap)
{
    MF_TRY MF_NEED(ctx) MF_MODEL(ctx, i) MF_OWNED(m)
    MaskFusion* o = ctx->mf.get();
    if (level < 0 || level > 2) { mf_set_error("level out of range"); return -2; }
    int Pl = (o->W >> level) * (o->H >> level);
    planarOut(o, m->vmapG[level], Pl, vmap);
    planarOut(o, m->nmapG[level], Pl, nmap);
    return 0;
    MF_CATCH(-1)
}
extern "C" int mf_download_index_map(mf_context* ctx, int i, uint32_t* idx, float* vc, float* ct, float* nr)
{
    MF_TRY MF_NEED(ctx) MF_MODEL(ctx, i) MF_OWNED(m)
    MaskFusion* o = ctx->mf.get();
    m->flushIndex();
    d2h(o, idx, m->idx.p, o->P); d2h(o, vc, m->vertConf.p, o->P); d2h(o, ct, m->colorTime.p, o->P); d2h(o, nr, m->normRad.p, o->P);
    o->sync(); return 0;
    MF_CATCH(-1)
}
extern "C" int mf_download_prediction(mf_context* ctx, int i, uint8_t* image4, float* vc, float* nr, uint16_t* time)
{
    MF_TRY MF_NEED(ctx) MF_MODEL(ctx, i) MF_OWNED(m)
    MaskFusion* o = ctx->mf.get();
    d2h(o, image4, m->splatImage.p, o->P); d2h(o, vc, m->splatVertex.p, o->P); d2h(o, nr, m->splatNormal.p, o->P); d2h(o, time, m->splatTime.p, o->P);
    o->sync(); return 0;
    MF_CATCH(-1)
}
extern "C" int mf_download_fill_in(mf_context* ctx, int i, uint8_t* image4, float* v4, float* n4)
{
    MF_TRY MF_NEED(ctx) MF_MODEL(ctx, i) MF_OWNED(m)
    MaskFusion* o = ctx->mf.get();
    if (!m->fillIn) { mf_set_error("model has no fill-in textures"); return -5; }
    d2h(o, image4, m->fillImage.p, o->P); d2h(o, v4, m->fillVertex.p, o->P); d2h(o, n4, m->fillNormal.p, o->P);
    o->sync(); return 0;
    MF_CATCH(-1)
}
extern "C" int mf_download_association(mf_context* ctx, int i, uint8_t* flag, uint32_t* best, float* meas12)
{
    MF_TRY MF_NEED(ctx) MF_MODEL(ctx, i) MF_OWNED(m)
    MaskFusion* o = ctx->mf.get();
    d2h(o, flag, m->aflag.p, o->P); d2h(o, best, m->abest.p, o->P);
    if (meas12) {
        DevBuf<float4> tmp; tmp.alloc((size_t)o->P * 3);
        launch_planes_to_aos(SurfelPlanes{m->meas[0].p, m->meas[1].p, m->meas[2].p}, (uint32_t)o->P, tmp, o->on());
        cudaCheck(cudaMemcpyAsync(meas12, tmp.p, (size_t)o->P * 48, cudaMemcpyDeviceToHost, o->stream), "D2H");
        o->sync();
    }
    o->sync(); return 0;
    MF_CATCH(-1)
}
extern "C" int mf_download_track_stats(mf_context* ctx, int i, double* A36, double* b6, float* err6)
{
    MF_TRY MF_NEED(ctx) MF_MODEL(ctx, i) MF_OWNED(m)
    MaskFusion* o = ctx->mf.get();
    TrackState st;
    cudaCheck(cudaMemcpyAsync(&st, m->trackState.p, sizeof st, cudaMemcpyDeviceToHost, o->stream), "D2H");
    o->sync();
    if (A36) memcpy(A36, st.lastA, sizeof st.lastA);
    if (b6) memcpy(b6, st.lastb, sizeof st.lastb);
    if (err6) { err6[0] = st.lastICPError; err6[1] = st.lastICPCount; err6[2] = st.lastRGBError; err6[3] = st.lastRGBCount; err6[4] = st.lastSO3Error; err6[5] = st.lastSO3Count; }
    return 0;
    MF_CATCH(-1)
}
extern "C" int mf_download_edge_map(mf_context* ctx, float* edge, uint8_t* binary)
{
    MF_TRY MF_NEED(ctx)
    MaskFusion* o = ctx->mf.get();
    o->edgeMaps();
    d2h(o, edge, o->edgeMap.p, o->P); d2h(o, binary, o->edgeInv.p, o->P);
    o->sync(); return 0;
    MF_CATCH(-1)
}

// test hook: the two morphological closes of the segmentation on a caller-given image (host, W x H of the context, in place).
//   ellipse != 0: gray-level close with OpenCV's elliptic element (mask-id image, MfSegmentation.cpp:424-426)
//   ellipse == 0: the binary close of the edge map (dilate_Kernel / erode_Kernel, segmentation.cu:217-255, host :334-354); `inverted` (may be
//                 NULL) receives 255 - result like MfSegmentation.cpp:208
extern "C" int mf_morph_close(mf_context* ctx, uint8_t* image, int radius, int iterations, int ellipse, uint8_t* inverted)
{
    MF_TRY MF_NEED(ctx)
    if (!image || radius < 0 || iterations < 0) { mf_set_error("morph_close: bad arguments"); return -3; }
    MaskFusion* o = ctx->mf.get();
    DevBuf<uint8_t> a, b, c; a.alloc(o->P); b.alloc(o->P); c.alloc(o->P);
    cudaCheck(cudaMemcpyAsync(a.p, image, o->P, cudaMemcpyHostToDevice, o->stream), "H2D");
    if (ellipse) launch_morph_close_ellipse(a, b, o->W, o->H, radius, iterations, nullptr, o->on());
    else launch_morph_close_invert(a, b, o->W, o->H, radius, iterations, c, o->on());
    d2h(o, image, a.p, o->P);
    if (inverted && !ellipse) d2h(o, inverted, c.p, o->P);
    o->sync(); return 0;
    MF_CATCH(-1)
}

// test hook: the segmentation after the edge map (MaskFusion::segmentEdges, the code the frame path runs) on caller-given inputs and a
// caller-given model list.  The inputs go into the buffers the frame path reads (the inverted edge map, the current slot's raw depth, mask
// and header, the projected-ID image); the segmentation is written to a buffer of the call, so the context's textureMask is untouched,
// and no FrameResult is left for the next processFrame to apply.  On purpose the call advances the state that persists across frames
// like the members of the reference class: the person ignore map and maskToID.  projected_ids must hold model ids (or 0), as the
// global projection gives them.
extern "C" int mf_debug_segment(mf_context* ctx, const uint8_t* edges_inv, const float* depth, const uint8_t* mask, int n_masks,
                                const int32_t* class_ids, const uint8_t* projected_ids, int n_models, const uint8_t* model_ids,
                                const int32_t* model_class_ids, int next_model_id, int allow_new, uint8_t* segmentation_out,
                                int32_t* labels_out, int32_t* result3_out)
{
    MF_TRY MF_NEED(ctx)
    MF_UNQUEUED(ctx, "debug_segment")
    MaskFusion* o = ctx->mf.get();
    if (!o->cfg.enableMultipleModels) { mf_set_error("not a multi-model context"); return -5; }
    if (n_masks < 0 || n_masks > 256 || n_models < 1 || n_models > MF_MAX_MODELS - 1 || next_model_id < 0 || next_model_id > 255) {
        mf_set_error("debug_segment: need n_masks in 0..256, n_models in 1..63 and next_model_id in 0..255"); return -3;
    }
    if (!edges_inv || !depth || !projected_ids || !model_ids || !model_class_ids || !segmentation_out || (n_masks && (!mask || !class_ids))) {
        mf_set_error("debug_segment: null input or output"); return -3;
    }
    bool isModel[256] = {};
    for (int i = 0; i < n_models; ++i) isModel[model_ids[i]] = true;
    for (int i = 0; i < o->P; ++i) {
        if (projected_ids[i] && !isModel[projected_ids[i]]) { mf_set_error("debug_segment: projected_ids holds an id that is no model's"); return -3; }
        if (n_masks && mask[i] >= n_masks) { mf_set_error("debug_segment: a mask value is not below n_masks"); return -3; }
    }
    o->waitHandoff(o->stream);                                      // a detector's hand-off into the current slot lands before ours
    SegModels sm; memset(&sm, 0, sizeof sm);
    sm.n = n_models; sm.nextID = (unsigned char)next_model_id;
    for (int i = 0; i < n_models; ++i) { sm.id[i] = model_ids[i]; sm.classID[i] = model_class_ids[i]; }
    FrameHdr h; memset(&h, 0, sizeof h);
    h.nMasks = n_masks; h.maskGiven = n_masks > 0;
    for (int i = 0; i < n_masks; ++i) h.classIDs[i] = class_ids[i];
    const size_t P = (size_t)o->P;
    cudaCheck(cudaMemcpyAsync(o->edgeInv.p, edges_inv, P, cudaMemcpyHostToDevice, o->stream), "H2D");
    cudaCheck(cudaMemcpyAsync(o->depthRaw, depth, P * sizeof(float), cudaMemcpyHostToDevice, o->stream), "H2D");
    if (n_masks) cudaCheck(cudaMemcpyAsync(o->frameMask, mask, P, cudaMemcpyHostToDevice, o->stream), "H2D");
    cudaCheck(cudaMemcpyAsync(o->projectedIDs.p, projected_ids, P, cudaMemcpyHostToDevice, o->stream), "H2D");
    launch_frame_header(h, o->dHdr, o->on());
    DevBuf<uint8_t> seg; seg.alloc(P);
    o->segTables(sm);
    o->segmentEdges(sm, allow_new != 0, seg);
    FrameResult r;
    d2h(o, segmentation_out, seg.p, P);
    d2h(o, labels_out, o->ccLabB.p, P);
    cudaCheck(cudaMemcpyAsync(&r, o->dRes.p, sizeof r, cudaMemcpyDeviceToHost, o->stream), "D2H");
    o->sync();
    if (result3_out) { result3_out[0] = r.hasNewLabel; result3_out[1] = r.newClassID; result3_out[2] = r.nComponents; }
    return 0;
    MF_CATCH(-1)
}

// Mask R-CNN backbone on the frame path: every k-th processFrame enqueues mold_inputs + the ResNet-101-FPN forward of `backbone`
// (mf_backbone_create) on the backbone's own stream (MaskRCNN::executeSequential is called from MfSegmentation.cpp:130). NULL detaches.
extern "C" int mf_attach_backbone(mf_context* ctx, void* backbone, int every_k)
{
    MF_TRY MF_NEED(ctx)
    ctx->mf->attachBackbone((mf_backbone*)backbone, every_k); return 0;
    MF_CATCH(-1)
}

// Mask R-CNN detector on the frame path (MfSegmentation.cpp:128-131, MaskRCNN.cpp:98-151): the masks of segmentation frames that the caller
// gives none come from `detector` every k-th tick.  NULL detaches (after the last hand-off has landed).
extern "C" int mf_attach_detector(mf_context* ctx, mf_detector* detector, int every_k)
{
    MF_TRY MF_NEED(ctx)
    ctx->mf->attachDetector(detector, every_k); return 0;
    MF_CATCH(-1)
}
// FrameData::mask / classIDs as segmentation read them on the last frame (replaces the reference's WRITE_MASK_FILES dump)
extern "C" int mf_download_frame_masks(mf_context* ctx, uint8_t* mask, int32_t* class_ids_256, int* n_masks)
{
    MF_TRY MF_NEED(ctx)
    MaskFusion* o = ctx->mf.get();
    if (!o->cfg.enableMultipleModels) { mf_set_error("not a multi-model context"); return -5; }
    // a queued frame popped by an in_pose call was detected at push time but does not segment, so nothing has waited for its hand-off yet
    o->waitHandoff(o->stream);
    FrameHdr h;
    cudaCheck(cudaMemcpyAsync(&h, o->dHdr, sizeof h, cudaMemcpyDeviceToHost, o->stream), "D2H");
    d2h(o, mask, o->frameMask, o->P);
    o->sync();
    if (mask && h.nMasks == 0) memset(mask, 0, o->P);            // a frame without masks: the set's mask bytes are stale
    if (class_ids_256) memcpy(class_ids_256, h.classIDs, sizeof h.classIDs);
    if (n_masks) *n_masks = h.nMasks;
    return 0;
    MF_CATCH(-1)
}

// stage clock of the last tracking launch: (tag, SM clock) pairs; 0 unless the library was built with -DMF_TRACK_TIMING (A/B builds)
extern "C" int mf_debug_track_timing(int64_t* out, int cap) { return debug_track_timing((long long*)out, cap); }

extern "C" int mf_set_frame_classes(mf_context* ctx, const int32_t* class_ids, int n)
{
    MF_TRY MF_NEED(ctx)
    if (n < 0 || n > 256) { mf_set_error("class id list must have 0..256 entries"); return -3; }
    ctx->mf->setFrameClasses(class_ids, n);
    return 0;
    MF_CATCH(-1)
}
extern "C" int mf_download_segmentation(mf_context* ctx, uint8_t* mask, uint8_t* projected_ids)
{
    MF_TRY MF_NEED(ctx)
    MaskFusion* o = ctx->mf.get();
    d2h(o, mask, o->mask.p, o->P);
    if (projected_ids) { if (!o->projectedIDs.p) { mf_set_error("not a multi-model context"); return -5; } d2h(o, projected_ids, o->projectedIDs.p, o->P); }
    o->sync(); return 0;
    MF_CATCH(-1)
}
// ---- object-sharded mode (SURVEY 8e) ----
extern "C" int mf_shard_configure(mf_context* ctx, int rank, int world) { MF_TRY MF_NEED(ctx) ctx->mf->configureShard(rank, world); return 0; MF_CATCH(-1) }
extern "C" int mf_shard_frame_begin(mf_context* ctx, const void* rgb, const void* depth, int64_t ts, const void* mask, int on_device)
{
    MF_TRY MF_NEED(ctx)
    if (!rgb || !depth || ts < 0) { mf_set_error("frame_begin: rgb/depth must be non-null and timestamp >= 0"); return -3; }
    ctx->mf->frameBegin((const uint8_t*)rgb, (const float*)depth, ts, (const uint8_t*)mask, nullptr, false, on_device != 0);
    return 0;
    MF_CATCH(-1)
}
extern "C" int mf_shard_get_poses(mf_context* ctx, float* out, int capacity_models)
{
    MF_TRY MF_NEED(ctx)
    if (capacity_models < MF_MAX_MODELS) { mf_set_error("get_poses: the buffer must hold 64 rows of 32 floats"); return -2; }
    ctx->mf->getShardPoses(out);
    return (int)ctx->mf->models.size();
    MF_CATCH(-1)
}
extern "C" int mf_shard_unique_id(uint8_t* out128)
{
    MF_TRY
    if (!out128) { mf_set_error("null buffer"); return -1; }
    shardUniqueId(out128); return 0;
    MF_CATCH(-1)
}
extern "C" int mf_shard_comm_init(mf_context* ctx, const uint8_t* id128, int rank, int world)
{
    MF_TRY MF_NEED(ctx)
    if (!id128) { mf_set_error("null id"); return -1; }
    ctx->mf->initShardComm(id128, rank, world); return 0;
    MF_CATCH(-1)
}
extern "C" int mf_shard_process_frame(mf_context* ctx, const uint8_t* rgb, const float* depth, int64_t ts, const uint8_t* mask, const int32_t* class_ids,
                                      int n_class_ids, float weight_multiplier, int inputs_on_device)
{
    MF_TRY MF_NEED(ctx)
    MaskFusion* o = ctx->mf.get();
    if (!o->shardNccl) { mf_set_error("mf_shard_process_frame needs a communicator (mf_shard_comm_init)"); return -2; }
    if (o->rank == 0) {
        if (!rgb || !depth || ts < 0) { mf_set_error("processFrame: rgb/depth must be non-null and timestamp >= 0 on the loader rank"); return -3; }
        if (n_class_ids < 0 || n_class_ids > 256) { mf_set_error("class id list must have 0..256 entries"); return -3; }
        o->setFrameClasses(class_ids, class_ids ? n_class_ids : 0);
    }
    o->processFrame(rgb, depth, ts, mask, nullptr, weight_multiplier, false, inputs_on_device != 0);
    return 0;
    MF_CATCH(-1)
}
extern "C" int mf_shard_stats(mf_context* ctx, int64_t* out4)
{
    MF_TRY
    if (!ctx || !ctx->mf || !out4) { mf_set_error("null argument"); return -1; }
    MaskFusion* o = ctx->mf.get();
    out4[0] = (int64_t)o->shard.bytesMoved; out4[1] = o->shard.calls; out4[2] = o->shardNccl ? o->shard.world : 0; out4[3] = o->shard.version;
    return 0;
    MF_CATCH(-1)
}
extern "C" int mf_shard_set_poses(mf_context* ctx, const float* gathered) { MF_TRY MF_NEED(ctx) ctx->mf->setShardPoses(gathered); return 0; MF_CATCH(-1) }
extern "C" int mf_shard_project(mf_context* ctx) { MF_TRY MF_NEED(ctx) ctx->mf->frameProject(); return 0; MF_CATCH(-1) }
extern "C" void* mf_shard_projection_keys(mf_context* ctx) { if (!ctx || !ctx->mf) return nullptr; return ctx->mf->projKeys.p; }
extern "C" int mf_shard_frame_end(mf_context* ctx, float weight_multiplier) { MF_TRY MF_NEED(ctx) ctx->mf->frameEnd(weight_multiplier); return 0; MF_CATCH(-1) }
// Mask R-CNN detector in the object-sharded mode: detection on detector_rank, its mask + header broadcast to every rank on detector frames
extern "C" int mf_shard_attach_detector(mf_context* ctx, mf_detector* detector, int every_k, int detector_rank)
{
    MF_TRY MF_NEED(ctx)
    ctx->mf->attachShardDetector(detector, every_k, detector_rank); return 0;
    MF_CATCH(-1)
}
extern "C" int mf_shard_frame_masks(mf_context* ctx, void** d_ptr, size_t* bytes)
{
    MF_TRY MF_NEED(ctx)
    if (!d_ptr || !bytes) { mf_set_error("frame_masks: null output"); return -3; }
    void* p = nullptr; size_t n = 0;
    if (!ctx->mf->shardFrameMasks(&p, &n)) return 0;
    *d_ptr = p; *bytes = n;
    return 1;
    MF_CATCH(-1)
}
extern "C" int mf_model_owner(mf_context* ctx, int i) { MF_TRY MF_NEED(ctx) MF_MODEL(ctx, i) return m->ownerRank; MF_CATCH(-1) }
extern "C" int mf_track_shares(int n_jobs, unsigned light_mask, int total_ctas, int ratio, int* shares)
{
    if (!shares || n_jobs < 1 || n_jobs > TRACK_MAX_JOBS || total_ctas < n_jobs) return -1;
    track_shares(n_jobs, light_mask, total_ctas, ratio, shares);
    return 0;
}
extern "C" int mf_shard_pick_owner(const int64_t* loads, int world) { if (!loads || world < 1 || world > 64) return -1; return MaskFusion::pickOwner(loads, world); }

extern "C" int mf_model_class_id(mf_context* ctx, int i) { MF_TRY MF_NEED(ctx) MF_MODEL(ctx, i) return m->classID; MF_CATCH(-1) }
extern "C" int mf_set_profiling(mf_context* ctx, int on)
{
    MF_TRY MF_NEED(ctx)
    ctx->mf->sync();
    Profiler& p = ctx->mf->rec.prof;
    p.on = on != 0; p.used = 0;
    if (on) p.acc.clear();
    return 0;
    MF_CATCH(-1)
}
extern "C" int mf_get_stage_times(mf_context* ctx, char* buf, int bufsize)
{
    MF_TRY MF_NEED(ctx)
    ctx->mf->sync();
    std::string out;
    char line[256];
    for (auto& kv : ctx->mf->rec.prof.acc) { snprintf(line, sizeof line, "%s %ld %.6f\n", kv.first.c_str(), kv.second.first, kv.second.second); out += line; }
    if ((int)out.size() + 1 > bufsize) { mf_set_error("buffer too small"); return -6; }
    memcpy(buf, out.c_str(), out.size() + 1);
    return (int)out.size();
    MF_CATCH(-1)
}
extern "C" int mf_debug_set_poses(mf_context* ctx, int i, const float* pose16, const float* last16)
{
    MF_TRY MF_NEED(ctx) MF_MODEL(ctx, i)
    m->pose = fromColMajor(pose16); m->lastPose = fromColMajor(last16);
    m->pushPose();
    return 0;
    MF_CATCH(-1)
}
// ======================================================================================
// .klg reader / writer (GUI/Tools/KlgLogReader.cpp:29-113): raw or zlib-compressed depth, raw or JPEG-compressed colour
// (decoded by mf_jpeg.cu, a restatement of libjpeg's default decode path).
// ======================================================================================
struct mf_klg {
    FILE* fp = nullptr; int W, H, numFrames, currentFrame; int flip;
    std::vector<unsigned char> dbuf, rbuf, dec;
    ~mf_klg() { if (fp) fclose(fp); }
};
extern "C" mf_klg* mf_klg_open(const char* path, int width, int height, int flip_colors)
{
    MF_TRY
    if (!path) { mf_set_error("mf_klg_open: null path"); return nullptr; }
    if (width <= 0 || height <= 0 || width > 16384 || height > 16384) { mf_set_error("mf_klg_open: width/height must be in 1..16384"); return nullptr; }
    std::unique_ptr<mf_klg> k(new mf_klg);
    k->fp = fopen(path, "rb");
    int32_t n = 0;
    if (!k->fp || !fread(&n, sizeof(int32_t), 1, k->fp)) { mf_set_error(std::string("Could not open log-file: ") + path); return nullptr; }
    k->W = width; k->H = height; k->numFrames = n; k->currentFrame = 0; k->flip = flip_colors;
    size_t P = (size_t)width * height;
    k->dbuf.resize(P * 2 + 1024); k->rbuf.resize(P * 3 + 1024); k->dec.resize(P * 2);
    return k.release();
    MF_CATCH(nullptr)
}
extern "C" int mf_klg_num_frames(mf_klg* k) { return k ? k->numFrames : -1; }
extern "C" int mf_klg_has_more(mf_klg* k) { return k ? (k->currentFrame + 1 < k->numFrames) : 0; }   // KlgLogReader.cpp:113 (N11)
extern "C" int mf_klg_get_next(mf_klg* k, uint8_t* rgb, float* depth, int64_t* timestamp)
{
    MF_TRY
    if (!k || !rgb || !depth) { mf_set_error("mf_klg_get_next: null reader or output buffer"); return -1; }
    const size_t P = (size_t)k->W * k->H;
    int64_t ts; int32_t dsz, rsz;
    if (!fread(&ts, sizeof ts, 1, k->fp) || !fread(&dsz, sizeof dsz, 1, k->fp) || !fread(&rsz, sizeof rsz, 1, k->fp)) { mf_set_error("klg: truncated frame header"); return -2; }
    if (dsz < 0 || rsz < 0 || (size_t)dsz > k->dbuf.size() || (size_t)rsz > k->rbuf.size()) { mf_set_error("klg: implausible frame sizes"); return -3; }
    if (dsz && !fread(k->dbuf.data(), dsz, 1, k->fp)) { mf_set_error("klg: truncated depth"); return -2; }
    if (rsz > 0 && !fread(k->rbuf.data(), rsz, 1, k->fp)) { mf_set_error("klg: truncated rgb"); return -2; }
    const uint16_t* d16 = (const uint16_t*)k->dbuf.data();
    if ((size_t)dsz != P * 2) {
        unsigned long len = (unsigned long)(P * 2);
        if (uncompress(k->dec.data(), &len, k->dbuf.data(), (unsigned long)dsz) != Z_OK) { mf_set_error("klg: zlib depth decode failed"); return -4; }
        d16 = (const uint16_t*)k->dec.data();
    }
    for (size_t i = 0; i < P; ++i) depth[i] = (float)((double)d16[i] * 0.001);         // convertTo(CV_32FC1, 0.001), KlgLogReader.cpp:68-70
    if (rsz > 0) {
        if ((size_t)rsz != P * 3) {
            // JPEG colour (KlgLogReader.cpp:72-79 -> JPEGLoader::readData): libjpeg's RGB rows with R and B exchanged (JPEGLoader.h:72-81)
            int jw = 0, jh = 0; std::vector<uint8_t> dec; std::string err;
            if (!mfb::decodeJPEG(k->rbuf.data(), (size_t)rsz, jw, jh, dec, err)) { mf_set_error("klg: " + err); return -5; }
            if (jw != k->W || jh != k->H) { mf_set_error("klg: JPEG frame size differs from the reader's resolution"); return -5; }
            for (size_t i = 0; i < P * 3; i += 3) { rgb[i] = dec[i + 2]; rgb[i + 1] = dec[i + 1]; rgb[i + 2] = dec[i]; }
        } else memcpy(rgb, k->rbuf.data(), P * 3);
    } else memset(rgb, 0, P * 3);
    if (k->flip) for (size_t i = 0; i < P * 3; i += 3) { uint8_t t = rgb[i]; rgb[i] = rgb[i + 2]; rgb[i + 2] = t; }
    if (timestamp) *timestamp = ts;
    k->currentFrame++;
    return 0;
    MF_CATCH(-6)
}
extern "C" void mf_klg_close(mf_klg* k) { delete k; }
extern "C" int mf_klg_write(const char* path, int width, int height, int num_frames, const int64_t* timestamps, const uint16_t* depth_mm, const uint8_t* rgb)
{
    MF_TRY
    if (!path || width <= 0 || height <= 0 || num_frames < 0 || (num_frames > 0 && (!timestamps || !depth_mm || !rgb))) { mf_set_error("mf_klg_write: bad arguments"); return -1; }
    FILE* fp = fopen(path, "wb");
    if (!fp) { mf_set_error(std::string("cannot write ") + path); return -1; }
    const size_t P = (size_t)width * height;
    int32_t n = num_frames, dsz = (int32_t)(P * 2), rsz = (int32_t)(P * 3);
    fwrite(&n, sizeof n, 1, fp);
    for (int f = 0; f < num_frames; ++f) {
        fwrite(&timestamps[f], sizeof(int64_t), 1, fp);
        fwrite(&dsz, sizeof dsz, 1, fp); fwrite(&rsz, sizeof rsz, 1, fp);
        fwrite(depth_mm + (size_t)f * P, 2, P, fp);
        fwrite(rgb + (size_t)f * P * 3, 1, P * 3, fp);
    }
    fclose(fp);
    return 0;
    MF_CATCH(-1)
}
