// mf_kernels.h -- host-callable launchers of the sm_90a kernels and the device-side
// structures they share with the host classes (mf_host.cu).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <string.h>
#include <exception>
#include <mutex>
#include <string>
#include <utility>
#include <vector>
#include "mf_common.cuh"

struct mf_backbone;
struct mf_rpn;
struct mf_detector;

// the calling thread's error message, which mf_last_error() returns (mf_capi.cu); every C ABI entry point reports through it
void mf_set_error(const std::string& msg);

// the guard of every extern "C" function that can fail: nothing thrown below it unwinds into the caller's frames.  A CudaError's text is
// stored after `cudaPrefix`, any other exception as "<entry point>: <what()>"; the function then returns `ret`.
#define MF_TRY try {
#define MF_CATCH_AS(ret, cudaPrefix)                                                                          \
    } catch (const mfb::CudaError& e) { mf_set_error(cudaPrefix + e.what); return ret; }                      \
    catch (const std::exception& e) { mf_set_error(std::string(__func__) + ": " + e.what()); return ret; }     \
    catch (...) { mf_set_error(std::string(__func__) + ": unknown error"); return ret; }
#define MF_CATCH(ret) MF_CATCH_AS(ret, std::string())

namespace mfb {

struct SurfelPlanes { float4* pos; float4* col; float4* nrm; };

struct CudaError { std::string what; };
void cudaCheck(cudaError_t e, const char* where);        // throws CudaError

// Owners of the CUDA resources a context holds: empty when constructed, acquired by an explicit call, released by the destructor (errors
// ignored there), so a throw anywhere in a constructor unwinds what it acquired.  Acquisition is not the owner's constructor because a
// context's members are constructed before it selects its device.
template <typename T>
struct DevBuf {
    T* p = nullptr; size_t n = 0;
    DevBuf() {}
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { if (p) cudaFree(p); }
    void alloc(size_t count) { if (p) cudaFree(p); p = nullptr; n = 0; if (count) cudaCheck(cudaMalloc((void**)&p, count * sizeof(T)), "cudaMalloc"); n = count; }
    void zero(cudaStream_t s) { if (n) cudaCheck(cudaMemsetAsync(p, 0, n * sizeof(T), s), "memset"); }
    operator T*() const { return p; }
};
// pinned host memory, zero-filled by alloc
template <typename T>
struct HostBuf {
    T* p = nullptr;
    HostBuf() {}
    HostBuf(const HostBuf&) = delete;
    HostBuf& operator=(const HostBuf&) = delete;
    ~HostBuf() { if (p) cudaFreeHost(p); }
    void alloc(size_t count) { if (p) cudaFreeHost(p); p = nullptr; cudaCheck(cudaMallocHost((void**)&p, count * sizeof(T)), "cudaMallocHost"); memset(p, 0, count * sizeof(T)); }
    operator T*() const { return p; }
};
struct Event {
    cudaEvent_t e = nullptr;
    Event() {}
    Event(Event&& o) noexcept : e(o.e) { o.e = nullptr; }
    Event(const Event&) = delete;
    Event& operator=(const Event&) = delete;
    ~Event() { if (e) cudaEventDestroy(e); }
    void create(unsigned flags = cudaEventDisableTiming) { if (e) cudaEventDestroy(e); e = nullptr; cudaEvent_t h; cudaCheck(cudaEventCreateWithFlags(&h, flags), "cudaEventCreate"); e = h; }
    operator cudaEvent_t() const { return e; }
};
struct Stream {
    cudaStream_t s = nullptr;
    Stream() {}
    Stream(const Stream&) = delete;
    Stream& operator=(const Stream&) = delete;
    ~Stream() { if (s) cudaStreamDestroy(s); }
    void create() { if (s) cudaStreamDestroy(s); s = nullptr; cudaStream_t h; cudaCheck(cudaStreamCreateWithFlags(&h, cudaStreamNonBlocking), "cudaStreamCreate"); s = h; }
    operator cudaStream_t() const { return s; }
};

// A value that belongs to a device (an SM count, an occupancy, a kernel attribute set on it): `make(device)` runs the first time get() is
// called with that device current, from whichever thread gets there first, and its result is kept for the process.  If `make` throws,
// the exception reaches that caller and the next get() on the device runs it again.
template <typename T>
class PerDevice {
public:
    explicit PerDevice(T (*make)(int device)) : make_(make) {}
    PerDevice(const PerDevice&) = delete;
    PerDevice& operator=(const PerDevice&) = delete;
    const T& get()
    {
        int dev = 0;
        cudaCheck(cudaGetDevice(&dev), "cudaGetDevice");
        if (dev < 0 || dev >= kMaxDevices) throw CudaError{"device ordinal above 63"};
        std::call_once(once_[dev], [&] { value_[dev] = make_(dev); });
        return value_[dev];
    }
private:
    static constexpr int kMaxDevices = 64;
    T (*make_)(int);
    std::once_flag once_[kMaxDevices];
    T value_[kMaxDevices] = {};
};

// photometric correspondence record (reference: DataTerm, Core/Cuda/types.cuh:75-81)
struct DataTerm { short2 zero; short2 one; float diff; int valid; };

#define TRACK_MAX_JOBS 32        // tracked models of one batched launch (configs[4]: 16 objects + background)
#define TRACK_MAX_BLOCKS 1024
struct TrackPoses { float p[TRACK_MAX_JOBS][16]; };

// Pose of one model as the kernels see it: DEVICE resident, so that the passes after tracking (index map, association,
// fusion, clean, splat) are enqueued without waiting for the tracked pose on the host.  Written by the tracking kernel's
// epilogue or by k_set_pose (host-driven poses); both run the same derivePose().
//   pose  : Model::pose, camera -> model frame, row-major [R|t]
//   tinv  : pose.inverse() as [R^T | -R^T t] (rule R-INV)
//   fusionW : Model::computeFusionWeight(1.0), Model.cpp:449-464 (the caller's weightMultiplier is applied by the kernel)
struct DevPose { Rt pose; Rt tinv; float fusionW; float pad[7]; };

#ifdef __CUDACC__
// Model::rodrigues2 (Model.cpp:890-932) without the SVD re-orthonormalisation (rule R-SVD, DESIGN.md); R row-major 3x3
__device__ inline void rodrigues2Dev(const float* R, float* out)
{
    double rx = R[7] - R[5], ry = R[2] - R[6], rz = R[3] - R[1];
    double s = sqrt((rx * rx + ry * ry + rz * rz) * 0.25);
    double c = ((double)(R[0] + R[4] + R[8]) - 1) * 0.5;
    c = c > 1. ? 1. : c < -1. ? -1. : c;
    double theta = acos(c);
    if (s < 1e-5) {
        double t;
        if (c > 0) rx = ry = rz = 0;
        else {
            t = (R[0] + 1) * 0.5; rx = sqrt(t > 0 ? t : 0.0);
            t = (R[4] + 1) * 0.5; ry = sqrt(t > 0 ? t : 0.0) * (R[1] < 0 ? -1.0 : 1.0);
            t = (R[8] + 1) * 0.5; rz = sqrt(t > 0 ? t : 0.0) * (R[2] < 0 ? -1.0 : 1.0);
            if (fabs(rx) < fabs(ry) && fabs(rx) < fabs(rz) && (R[5] > 0) != (ry * rz > 0)) rz = -rz;
            theta /= sqrt(rx * rx + ry * ry + rz * rz);
            rx *= theta; ry *= theta; rz *= theta;
        }
    } else {
        double vth = 1 / (2 * s); vth *= theta; rx *= vth; ry *= vth; rz *= vth;
    }
    out[0] = (float)rx; out[1] = (float)ry; out[2] = (float)rz;
}

// pose (row-major 4x4, rigid) + the pose before this frame's update -> everything the surfel passes read.
// One thread.  tinv: [R^T | -R^T t] in fp32 with the operation order of the host rule (R-INV);
// fusionW: max(1 - max(|t|, |rotation vector|) of (pose^-1 * lastPose) / 0.01, 0.5)  (Model.cpp:449-464)
__device__ inline void derivePose(DevPose* d, const float* m, const float* last)
{
    float inv[16];
    {
        const float R[9] = {m[0], m[1], m[2], m[4], m[5], m[6], m[8], m[9], m[10]}, t[3] = {m[3], m[7], m[11]};
        for (int r = 0; r < 3; ++r) {
            for (int c = 0; c < 3; ++c) inv[r * 4 + c] = R[c * 3 + r];
            inv[r * 4 + 3] = -((R[0 * 3 + r] * t[0] + R[1 * 3 + r] * t[1]) + R[2 * 3 + r] * t[2]);
        }
        inv[12] = 0.f; inv[13] = 0.f; inv[14] = 0.f; inv[15] = 1.f;
    }
    for (int k = 0; k < 12; ++k) { d->pose.m[k] = m[k]; d->tinv.m[k] = inv[k]; }
    // diff = pose^-1 * lastPose, full 4x4 product in the order of the host routine (s += A[r][k] * B[k][c], k = 0..3)
    float diff[16];
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) {
            float s = 0;
            for (int k = 0; k < 4; ++k) s += inv[r * 4 + k] * last[k * 4 + c];
            diff[r * 4 + c] = s;
        }
    const float R[9] = {diff[0], diff[1], diff[2], diff[4], diff[5], diff[6], diff[8], diff[9], diff[10]};
    float tn = sqrtf((diff[3] * diff[3] + diff[7] * diff[7]) + diff[11] * diff[11]);
    float rv[3]; rodrigues2Dev(R, rv);
    float rn = sqrtf((rv[0] * rv[0] + rv[1] * rv[1]) + rv[2] * rv[2]);
    float weighting = tn > rn ? tn : rn;
    const float largest = 0.01f, minWeight = 0.5f;
    if (weighting > largest) weighting = largest;
    float w = 1.0f - (weighting / largest);
    d->fusionW = w > minWeight ? w : minWeight;
}
#endif

// ---- device-resident frame bookkeeping of the multi-model schedule: nothing in a frame waits for the host ----
// FrameHdr: what the loader knows about the frame besides the images; in the object-sharded mode it is the tail of the broadcast
// frame packet, so the ranks that never saw the host inputs read it where the kernels read it: on the device.
// detectError: the attached detector's export rule failed on this frame (special_assignments[class_id] out of range), which then carries no masks
// maskGiven: the caller passed a mask with the frame; the detector's hand-off (k_frame_masks) then leaves mask and header alone.  It travels
// in the packet because a sharded run's detector rank may not be the rank that received the caller's inputs.
struct FrameHdr { long long timestamp; int nMasks; int detectError; int classIDs[256]; int maskGiven; };   // nMasks == 0: the frame carries no instance masks
// FrameResult: everything the host learns from a frame (one asynchronous copy behind the vote kernel; read at the START of the next
// frame): the spawn decision of MfSegmentation, which tracked models jumped > 0.2 m (MaskFusion.cpp:268-272), every model's pose,
// the header's detectError.
#define MF_MAX_MODELS 64
struct FrameResult {
    int hasNewLabel, newClassID, nMasks, nComponents; long long timestamp;
    int dead[MF_MAX_MODELS]; unsigned deadCount[MF_MAX_MODELS];
    float poses[MF_MAX_MODELS][32];                       // pose (row-major 4x4) | last incremental transform
    int detectError;
};
struct SegTables { unsigned char idToIndex[256], indexToId[256], isModel[256]; };
struct VoteParams {
    int nModels, allowNew, personClassID; unsigned minNew, maxNew; float minMaskModelOverlap; unsigned char nextModelID;
    int modelClass[MF_MAX_MODELS]; unsigned char modelID[MF_MAX_MODELS];
};
struct LifeModel { int tracked, owned, ownerRank, pad; DevPose* dpose; const float* trackOut; unsigned* count; float initialC2Winv[16]; };
struct LifeParams { int nModels, rank; LifeModel m[MF_MAX_MODELS]; };

// Gauss-Newton state of one tracked model; lives in device memory for the whole frame
struct TrackState {
    float Rprev[9], tprev[3], RprevInv[9];
    float Rcurr[9], tcurr[3];
    float trR[9], trT[3];
    double resultRt[16];
    double resultR[9], lastResultR[9];
    float R_lr[9];
    float so3LastError, so3LastCount; int so3Done;
    float krk[9], kt[3];
    float sigmaVal; int levelBreak;
    float lastICPError, lastICPCount, lastRGBError, lastRGBCount, lastSO3Error, lastSO3Count;
    double lastA[36], lastb[6];
    float out[40];
    unsigned ticket[4];
};

struct TrackJob {
    const float4* vmapC[3]; const float4* nmapC[3];        // frame maps (shared by all models)
    const uint8_t* nextImage[3]; const short2* nextGrad[3]; const uint8_t* rgbValid[3];
    const float4* vmapG[3]; const float4* nmapG[3];        // model maps in the model-global frame
    const float* lastDepth[3]; const uint8_t* lastImage[3];
    const uint8_t* lastNextImage2;
    const float4* cloud[3];
    DataTerm* corres[3];
    DevPose* dpose;       // initial pose in, tracked pose + derived quantities out
    TrackState* st;
    float* partial;       // 2 x (TRACK_MAX_BLOCKS / 2) rows of 32 x 16 bytes: per-CTA partial sums (fp64 value + flags), ping-pong between reductions
    const uint32_t* validBits[3];   // object models: one bit per model-map pixel, set where the model normal is valid (nullptr: not used)
};

int num_sms();                  // SMs of the current device

// Where a dense-pipeline launcher enqueues: the stream and the launch record of the context it works for (mf_host.h: the launch
// count of mf_kernel_launches and the stage timer).  A null record counts and times nothing.
struct LaunchRecord;
struct Enq {
    cudaStream_t s;
    LaunchRecord* rec;
    // profiling on: a CUDA event on `s`; the time until the next mark is attributed to `name` (nullptr: to no stage)
    void mark(const char* name) const;
    // after a launch: throws CudaError naming `kernel` if the runtime's last error is set, else counts the launch
    void launched(const void* kernel) const;
};
// the one launch of a kernel: mark (name non-null), launch on q.s, check, count (a null record: check only)
template <typename... P, typename... A>
inline void launch(const Enq& q, const char* name, void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, A&&... args)
{
    if (name) q.mark(name);
    kernel<<<grid, block, smem, q.s>>>(std::forward<A>(args)...);
    q.launched((const void*)kernel);
}

// ---- mf_cnn.cu ----
// The Mask R-CNN handles (backbone, RPN, detector) belong to no context: every kernel of theirs goes through launch() with Enq{stream,
// nullptr}, which checks the launch and throws, and counts and times nothing.  Below their extern "C" entry points everything throws
// CudaError; only the entry points turn it into a return code.
// D[M x N] = relu?(A[M x K] * B[N x K]^T + bias + residual), bf16 operands; conv3x3 = {Wimg, Himg, Cin}: A is an NHWC activation and the GEMM is
// the implicit 3x3/s1/p1 convolution; outF32: D is fp32 (no residual), else bf16.  Every shape refusal throws before the first driver call
void launch_gemm_bf16(const void* A, const void* B, const float* bias, const void* residual, void* out, int M, int N, int K, int relu, cudaStream_t s,
                      const int* conv3x3 = nullptr, bool outF32 = false);
// one convolution (NHWC bf16, weights [Cout][Kpad] in (ky, kx, cin) order) through the backbone's conv path: the implicit 3x3 GEMM where its
// geometry guard admits the shape, else im2col into `col` (Hout*Wout*Kpad bf16) + GEMM
void cnn_conv(const void* in, int Hin, int Win, int Cin, int Cout, int k, int stride, int pad, const void* W, const float* B, void* col, void* out, int relu,
              cudaStream_t s);
bool cnn_conv_implicit(int k, int stride, int pad, int Cin, int Hin, int Win);     // does cnn_conv take the implicit path (no im2col)?
// im2col of `nimg` stacked NHWC images (each padded on its own): A[(img, oy, ox)][(ky, kx, cin)], K zero-padded to Kpad
void launch_im2col(const void* in, int nimg, int Hin, int Win, int Cin, int Hout, int Wout, int k, int stride, int pad, int Kpad, void* col, cudaStream_t s);
// the letter-box rule of mf_backbone_mold (mould_image): a W x H image is resized by `scale` to newW x newH and placed at (offx, offy) of S x S
struct MoldGeom { float scale; int newW, newH, offx, offy; };
MoldGeom cnn_mold_geometry(int S, int W, int H);
// the handles' read-back: `rows` rows of `width` bytes, `pitch` bytes apart on the device (0: one block), packed into dst after `s` is
// drained.  dst NULL: nothing is copied
void cnn_read_back(cudaStream_t s, void* dst, const void* src, size_t width, size_t rows = 1, size_t pitch = 0);
// the backbone handle: its stream; its input buffer (where backbone_mold writes); level 0..3 = C2..C5, 4..8 = P2..P6 as a device pointer
// with dims (H, W, C), nullptr for another level; the letter-boxed input of a W x H RGBA8 device image (W, H > 0); the forward on d_input
cudaStream_t backbone_stream(mf_backbone* h);
const void* backbone_input(mf_backbone* h);
void* backbone_level(mf_backbone* h, int level, int* dims3);
void backbone_mold(mf_backbone* h, const void* d_rgba, int W, int H);
void backbone_forward(mf_backbone* h, const void* d_input);

// ---- mf_rpn.cu: the RPN handle, and what the detection heads read of it ----
void rpn_run(mf_rpn* h, int stages);              // MF_RPN_* bits, in order
// pyramid ROI Align of n boxes on bb's P2..P5, on bb's stream
void roi_align(mf_backbone* bb, const float* boxes, int n, int pool, void* out);
mf_backbone* rpn_backbone(mf_rpn* h);
const float* rpn_rois(mf_rpn* h);                 // [1000][4] proposals, zero padded
const void* rpn_pooled(mf_rpn* h);                // [1000][7][7][256] bf16

// ---- mf_weights.cu: the layer table of the three Mask R-CNN handles and their weights (seeded, or pretrained: safetensors, R-FOLD) ----
enum { MRCNN_BACKBONE, MRCNN_RPN, MRCNN_DETECTOR };
// layer i of a handle, in its table order: input channels, GEMM rows (output channels and zero rows), kernel side, stride, pad, GEMM K
// (kh * kw * Cin zero padded).  The weights are [rows x K], (ky, kx, cin) along K; the bias [rows]
struct LayerGeom { int cin, rows, k, stride, pad, K; };
int mrcnn_num_layers(int part);
LayerGeom mrcnn_layer(int part, int i);
// every table of one handle in one pool: fp32 master copies (bf16-representable) on the host, bf16 weights and fp32 biases on the device
struct WeightStore {
    int part;
    std::vector<size_t> wOff, bOff;               // layer i: first element of its table / bias (128-byte aligned in the pools)
    std::vector<float> hW, hB;
    DevBuf<__nv_bfloat16> dW;
    DevBuf<float> dB;
    // the seeded tables (one LCG stream, seed 0 taken as 1), uploaded on `s`; throws CudaError
    WeightStore(int part, unsigned seed, cudaStream_t s);
    // every layer read, checked and folded on the host, uploaded on `s` and complete on return; the tables change only on success.
    // Throws CudaError naming the file and the tensor, or the failed upload
    void load(const char* path, cudaStream_t s);
    void get(int i, float* w, float* b, int rows = -1) const;   // the first `rows` rows (-1: all) of layer i; NULL skips; throws on a bad i
    const __nv_bfloat16* w(int i) const { return dW.p + wOff[i]; }
    const float* b(int i) const { return dB.p + bOff[i]; }
};

// ---- mf_heads.cu: the detector on the frame path (mf_attach_detector) ----
cudaStream_t detector_stream(mf_detector* h);
void detector_reserve_image(mf_detector* h, int W, int H);     // id image sized for W x H once: detector_detect at W x H then never reallocates
void detector_run(mf_detector* h, int stages);                 // MF_DET_* bits, in order
// what MaskRCNN.execute() does on a W x H RGBA8 device image (4-byte aligned): mould, backbone, RPN and every head stage, on one stream
void detector_detect(mf_detector* h, const void* d_rgba, int W, int H);
// FrameData::mask / classIDs from the last id image (MaskRCNN.cpp:98-112, 147-151), enqueued on the detector's stream: the id image into
// `mask` (W x H of the last detect), hdr->nMasks = exported + 1, hdr->classIDs = {0, exported class ids...}.  The count and ids stay on the
// device.  A failed export rule gives nMasks = 0 and hdr->detectError = 1.
void detector_frame_masks(mf_detector* h, uint8_t* mask, FrameHdr* hdr);

// ---- mf_frame.cu ----
void launch_unpack_rgb(const uint8_t* rgb3, uchar4* out, int P, Enq q);
void launch_bilateral(const float* depth, float* out, int W, int H, Enq q);
// fused variants: two pyramid levels per launch; three levels of a per-pixel kernel per launch (blockIdx.z = level)
void launch_pyrdown2_f(const float* src, int sw, int sh, float* dst1, float* dst2, Enq q);
void launch_pyrdown2_u8(const uint8_t* src, int sw, int sh, uint8_t* dst1, uint8_t* dst2, Enq q);
void launch_pyrdown2_pair(const float* srcF, float* dstF1, float* dstF2, const uint8_t* srcU, uint8_t* dstU1, uint8_t* dstU2, int sw, int sh, Enq q);
void launch_vmap_nmap3(const float* const* depth, int W, int H, Cam cam, float cutoff, float4* const* vmap, float4* const* nmap, Enq q);
void launch_sobel3(const uint8_t* const* img, int W, int H, short2* const* grad, uint8_t* const* rgbValid, Enq q);
void launch_project_points3(const float* const* depth, int W, int H, Cam cam, float4* const* cloud, Enq q);
void launch_intensity(const uchar4* img, int P, uint8_t* out, Enq q);
void launch_intensity_select(const uchar4* imgPred, const uchar4* imgFill, const uint32_t* nonBlack, float denom, int forceFill, int P, uint8_t* out, Enq q);
float track_min_scale(int level);          // gradient-magnitude gate of the photometric term at a pyramid level (RGBDOdometry.cpp:44-49)
void launch_model_maps(const float4* srcVp, const float4* srcNp, const float4* srcVf, const float4* srcNf, const uint32_t* nonBlack, float denom,
                       int W, int H, const DevPose* dpose, float maxDepthRGB, float4* const* v, float4* const* n, float* depth0, Enq q);
void launch_valid_bits3(const float4* const* nmap, int W, int H, uint32_t* const* bits, Enq q);    // bit i of level l = !isnan(nmap[l][i].x)
void launch_map_to_planar(const float4* m, int P, float* out, Enq q);

// ---- mf_surfel.cu ----
void launch_fill_u32(uint32_t* p, uint32_t v, size_t n, Enq q);
void launch_fill_u64(uint64_t* p, uint64_t v, size_t n, Enq q);
void launch_set_pose(DevPose* d, const float* pose16, const float* lastPose16, Enq q);      // host-driven pose -> DevPose
void launch_predict_indices(const SurfelPlanes& sp, const uint32_t* count, const DevPose* dpose, Cam cam, int W, int H, float maxDepth, int time,
                            int timeDelta, uint64_t* key, uint32_t* idx, float4* vertConf, float4* colorTime, float4* normRad, float4* cleanTex, float cleanConf,
                            Enq q);
void launch_associate(const uchar4* rgb, const float* depthRaw, const float* depthFilt, const uint8_t* mask, const uint32_t* idx,
                      const float4* vertConf, const float4* normRad, const DevPose* dpose, Cam cam, int W, int H, float maxDepth, int time,
                      float weightMultiplier, uint8_t maskID, uint8_t* flag, uint32_t* best, float4* const* meas, uint32_t* slot, Enq q);
void launch_fuse_update(const uint8_t* flag, const uint32_t* best, float4* const* meas, uint32_t* slot, int P, int time,
                        const SurfelPlanes& sp, Enq q);
// index-map outputs of a Model::predictIndices that is carried out INSIDE the clean pass (one stream over the store instead of two)
// what the index-map window of Model::clean reads: the packed 16-byte texels (written by the index resolve for THIS call's time and
// confidence threshold) or, packed == nullptr, the index-map images themselves
struct CleanWindowImages { const float4* packed; const float4* vertConf; const float4* colorTime; const uint32_t* idx; };
struct IndexFused { uint64_t* key; uint32_t* idx; float4* vertConf; float4* colorTime; float4* normRad; float4* cleanTex; float maxDepth; };
// in-place ordered compaction of Model::clean (k_clean_compact): ticket (reset by the sums pass), one published-epoch word per 512-entry
// sub-block, the first sub-block that holds a removal (written by the scan), the epoch of this call (never 0, changes with every call)
struct CleanInPlace { uint32_t* ticket; uint32_t* loaded; uint32_t* firstMoved; uint32_t epoch; bool pingPong; };   // firstMoved[0..1]: first moved sub-block, number of sub-blocks; pingPong: copy into `dst` instead (same result)
void launch_clean(const SurfelPlanes& src, const SurfelPlanes& dst, const uint32_t* count, uint32_t* newCount, uint32_t capacity,
                  const uint8_t* aflag, float4* const* meas, const DevPose* dpose, Cam cam, int W, int H, int time, int timeDelta, float confThreshold,
                  float outlierCoeff, uint8_t maskID, const CleanWindowImages& win,
                  const float* depthFilt, const uint8_t* mask, uint8_t* keep, uint32_t* blockSums, uint32_t* cand, uint32_t* candCount, Enq q,
                  const CleanInPlace& inplace, const IndexFused* fused = nullptr);
void launch_combined_predict(const SurfelPlanes& sp, const uint32_t* count, const DevPose* dpose, Cam cam, int W, int H, float maxDepth,
                             float confThreshold, int time, int maxTime, int timeDelta, const float4* rayTab, uint64_t* key, uchar4* image, float4* vertexConf,
                             float4* normalRad, uint16_t* timeTex, int doFill, const float* depthFilt, const uchar4* rgb, int ptVN, int ptImg,
                             uchar4* fillImage, float4* fillVertex, float4* fillNormal, uint32_t* nonBlackSamples, Enq q, uint32_t capacity = 0);
void launch_ray_table(Cam cam, int W, int H, float4* tab, Enq q);      // pixel-centre viewing rays (combo_splat.frag:39-45), once per context
void launch_init_model(const uchar4* rgb, const float* depthRaw, const float* depthFilt, Cam cam, int W, int H, int time, float maxDepth,
                       uint8_t* fr, uint8_t* ff, uint32_t* sumR, uint32_t* sumF, uint32_t capacity, const SurfelPlanes& sp, uint32_t* count,
                       Enq q);
void launch_planes_to_aos(const SurfelPlanes& sp, uint32_t n, float4* out, Enq q);
void launch_aos_to_planes(const float4* in, uint32_t n, const SurfelPlanes& sp, Enq q);

// ---- mf_track.cu ----
void track_shares(int nJobs, unsigned lightMask, int totalCTAs, int ratio, int* G);   // CTAs per model of the persistent tracking grid
// epoch: the flag epoch of this launch's partial-row exchange, advanced by the caller for every launch on the same partial buffers, never
// a value whose << 6 is 0 (TrackJob::partial; mf_track.cu)
void launch_tracking(TrackJob* d_jobs, int nJobs, int W, int H, Cam cam, bool rgbOnly, float icpWeight,
                     bool pyramid, bool fastOdom, bool so3, unsigned epoch, Enq q, unsigned lightMask = false);
int debug_track_timing(long long* out, int cap);
void launch_icp_only(const float4* vmapC, const float4* nmapC, const float4* vmapG, const float4* nmapG, int W, int H, Cam cam,
                     const TrackPoses& pp, float* partial, unsigned* ticket, float* out29, Enq q);

// ---- mf_seg.cu ----
void launch_geometric_edges(const float4* vmap, const float4* nmap, int W, int H, float wD, float wC, float thr, float* edge, uint8_t* binary, Enq q);
void launch_morph_close_ellipse(uint8_t* data, uint8_t* buf, int W, int H, int radius, int iterations, const FrameHdr* onlyIfMasks, Enq q);   // MfSegmentation.cpp:424-426
void launch_morph_close_invert(uint8_t* data, uint8_t* buf, int W, int H, int radius, int iterations, uint8_t* inverted, Enq q);

}  // namespace mfb

namespace mfb {
// ---- mf_seg.cu: GPU segmentation tail + global projection resolve ----
void launch_cc(const uint8_t* img, int W, int H, int* L, int* dense, int* lab, int* area, int* box, uint32_t* counter, Enq q);   // box: left, top, right, bottom per component
void launch_remove_edges(int* labA, int* labB, const float* depth, const int* area, int W, int H, int iterations, Enq q);
void launch_seg_tables(const SegTables& t, uint8_t* idToIndex, uint8_t* indexToId, uint8_t* isModel, Enq q);
void launch_frame_header(const FrameHdr& h, FrameHdr* d, Enq q);                       // single-process path: the header by value
void launch_person_table(const FrameHdr* hdr, int personClassID, uint8_t* isPerson, Enq q);
void launch_clear_hist(const uint32_t* ccCounter, const FrameHdr* hdr, int nModels, int* compModel, int* compMask, Enq q);
void launch_seg_hist(const int* lab, const uint8_t* projID, const uint8_t* mask, int P, const uint8_t* idToIndex, int nModels, const FrameHdr* hdr,
                     int* compModel, int* compMask, Enq q);
void launch_component_map(const uint32_t* ccCounter, const int* area, const int* compModel, const int* compMask, int nModels, const FrameHdr* hdr,
                          const uint8_t* indexToId, int minMapped, int* mapToMask, int* absorb, int* maskPixels, Enq q);
void launch_vote(const FrameHdr* hdr, const VoteParams& vp, const int* maskPixels, const unsigned* maskOverlap, const uint32_t* ccCounter,
                 uint8_t* maskToID, FrameResult* res, Enq q);
void launch_seg_assign(const int* lab, const int* mapToMask, const uint8_t* ignore, int P, uint8_t* seg, Enq q);
void launch_mask_overlap(const uint8_t* seg, const uint8_t* projID, const uint8_t* idToIndex, const uint8_t* isModelId, int P, unsigned* maskOverlap, Enq q);
void launch_seg_final(const uint8_t* seg, const int* lab, const int* mapToMask, const int* absorb, const uint8_t* maskToID, const int* box, int P, int W,
                      uint8_t* out, Enq q);
void launch_apply_ignore(const uint8_t* mask, const uint8_t* isPerson, const FrameHdr* hdr, int P, uint8_t* ignore, uint8_t* edges, Enq q);
void launch_proj_resolve(uint64_t* key, int P, const uint8_t* indexToId, uint8_t* out, Enq q);
void launch_splat_project_only(const SurfelPlanes& sp, const uint32_t* count, const DevPose* dpose, Cam cam, int W, int H, float maxDepth, float confThreshold,
                               int time, int maxTime, int timeDelta, uint32_t drawBase, const float4* rayTab, uint64_t* key, Enq q, uint32_t capacity = 0);
}  // namespace mfb
