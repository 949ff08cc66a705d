// mf_heads.cu -- Mask R-CNN detection heads on the RPN's proposals (sm_90a): classifier, detection layer, mask head, unmould + id image.
//
// matterport mrcnn's inference graph with the COCO InferenceConfig (NUM_CLASSES 81), written from upstream memory (the source is not
// vendored; DESIGN §3c, rules R-SOFTMAX / R-DETNMS / R-UNMOLD / R-RESIZE / R-SIGMOID in §4):
//   fpn_classifier_graph   7x7 valid conv 256->1024 + ReLU ("FC1": one GEMM on the RPN's pooled [1000][7][7][256] in place, K = 12 544),
//                          1x1 conv 1024->1024 + ReLU ("FC2"), class logits (81) + box deltas (81 x 4) as ONE GEMM: 405 rows zero-padded
//                          to 448, fp32 epilogue.  BatchNorm is in inference mode and folded into the seeded weights, as in the backbone.
//   DetectionLayer         softmax, argmax class, class-specific deltas x BBOX_STD_DEV, apply_box_deltas_graph, clip to the letter-box
//                          window, keep class > 0 and score >= 0.7, per-class greedy NMS at IoU 0.3 (<= 100 per class), top 100 by score
//                          -> [100][6] y1 x1 y2 x2 class score, zero padded, and the count (on the device)
//   build_fpn_mask_graph   ROI Align at 14 on the 100 detection rows, 4 x (3x3 conv 256->256 + ReLU) as im2col + GEMM (the implicit 3x3
//                          path refuses 14-wide images), 2x2/s2 transposed conv as a GEMM with N = 4 x 256 (rows [roi][y][x][dy][dx][c]),
//                          1x1 conv 256->81 (padded to 128, fp32) on those rows in place, then each detection's own class + sigmoid
//                          -> [100][28][28] fp32
//   unmold_detections +    k_unmold (one thread) maps the detections to integer boxes of the original image and applies
//   generate_id_image      generate_id_image's export rule; k_paste (one thread per pixel) walks the exported detections from last to first
//                          and writes the first whose resized mask is >= 0.5 there -- no H x W x N mask stack
//   hand-off               k_frame_masks (mf_attach_detector): the id image, [0] + exported class ids and their count into a frame's
//                          FrameData::mask / classIDs (MaskRCNN.cpp:98-112), read from the device buffers above
// Every stage is enqueued on the backbone's stream and runs on the fixed upstream shapes (1000 ROIs, 100 detection rows); nothing waits
// for the host.  Everything after the GEMMs is IEEE fp32 (fp64 where R-UNMOLD / R-RESIZE say so) in a fixed operation order (this file is
// compiled -fmad=false) and is reproduced bit for bit by the numpy restatement in tests/heads_ref.py.
#include "mf_common.cuh"
#include "mf_boxes.cuh"
#include "mf_kernels.h"
#include "../../include/maskfusion_b200.h"
#include <cuda_bf16.h>
#include <algorithm>
#include <assert.h>
#include <math.h>
#include <string.h>
#include <string>
#include <vector>

namespace mfb {

constexpr int DET_ROIS = 1000, DET_MAX = 100, NCLS = 81, FC_N = 1024, POOL = 7, CH = 256, HEAD_N = 448;
constexpr int MPOOL = 14, MPIX = MPOOL * MPOOL, MASK = 28, MLOG_N = 128, MCONV_K = 9 * CH, SEL_N = 1024, EXPORT_CAP = 128;
constexpr float DET_MIN_CONFIDENCE = 0.7f, DET_NMS_THRESHOLD = 0.3f;

// the handle's layers in the order of its table (mf_weights.cu)
enum { L_FC1, L_FC2, L_HEAD, L_M1, L_M2, L_M3, L_M4, L_DECONV, L_MLOG, N_LAYERS };

struct ExportParams { double min_score; int n_filter, n_special; int filter[EXPORT_CAP], special[EXPORT_CAP]; };

// R-SOFTMAX + argmax + class-specific refinement of one ROI per thread -> candidate key (class, ~ord(score), roi) or ~0, refined box, score
__global__ void k_det_refine(const float4* __restrict__ rois, const float* __restrict__ logits, int lstride, const float* __restrict__ deltas,
                             int dstride, int n, float4 win, unsigned long long* __restrict__ keys, float4* __restrict__ boxes, float* __restrict__ scores)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float* l = logits + (size_t)i * lstride;
    float m = l[0];
    for (int c = 1; c < NCLS; ++c) m = l[c] > m ? l[c] : m;
    float sum = 0.0f;
    for (int c = 0; c < NCLS; ++c) sum = sum + det_expf(l[c] - m);
    int best = 0;
    float pbest = det_expf(l[0] - m) / sum;
    for (int c = 1; c < NCLS; ++c) {
        const float p = det_expf(l[c] - m) / sum;
        if (p > pbest) { best = c; pbest = p; }
    }
    const float* d = deltas + (size_t)i * dstride + 4 * best;
    const float4 b = decode_box(rois[i], make_float4(d[0], d[1], d[2], d[3]), win);
    const bool keep = best > 0 && pbest >= DET_MIN_CONFIDENCE;
    keys[i] = keep ? ((unsigned long long)best << 42) | ((unsigned long long)(~score_ord(pbest)) << 10) | (unsigned)i : ~0ull;
    boxes[i] = b;
    scores[i] = pbest;
}

// one CTA of 1024: sort the candidates on (class, ~ord(score), roi), per-class greedy NMS (warp w: classes w + 1, w + 33, ...), sort the
// survivors on (~ord(score), roi), write the first 100 as detections (zero padded), their boxes for the mask head's ROI Align, the count
__global__ void __launch_bounds__(SEL_N) k_det_select(const unsigned long long* __restrict__ keys, int n, const float4* __restrict__ boxes,
                                                      const float* __restrict__ scores, float* __restrict__ dets, float4* __restrict__ dboxes,
                                                      int* __restrict__ count)
{
    __shared__ unsigned long long sk[SEL_N];
    __shared__ int segStart[NCLS], segEnd[NCLS];
    __shared__ unsigned char supp[SEL_N], kept[SEL_N];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    sk[t] = t < n ? keys[t] : ~0ull;
    supp[t] = 0; kept[t] = 0;
    if (t < NCLS) { segStart[t] = 0; segEnd[t] = 0; }
    __syncthreads();
    cta_bitonic_sort(sk, SEL_N);
    const int cls = sk[t] == ~0ull ? -1 : (int)(sk[t] >> 42);
    if (cls > 0) {
        if (t == 0 || (int)(sk[t - 1] >> 42) != cls) segStart[cls] = t;
        if (t == SEL_N - 1 || sk[t + 1] == ~0ull || (int)(sk[t + 1] >> 42) != cls) segEnd[cls] = t + 1;
    }
    __syncthreads();
    for (int c = 1 + warp; c < NCLS; c += SEL_N / 32) {
        const int st = segStart[c], en = segEnd[c];
        int nk = 0;
        for (int i = st; i < en && nk < DET_MAX; ++i) {
            __syncwarp();
            if (supp[i]) continue;
            ++nk;
            if (lane == 0) kept[i] = 1;
            const float4 bi = boxes[sk[i] & 1023];
            for (int j = i + 1 + lane; j < en; j += 32)
                if (iou_tf(bi, boxes[sk[j] & 1023]) > DET_NMS_THRESHOLD) supp[j] = 1;
        }
    }
    __syncthreads();
    unsigned long long k2 = ~0ull;
    if (kept[t]) {
        const unsigned roi = (unsigned)(sk[t] & 1023);
        k2 = ((unsigned long long)(~score_ord(scores[roi])) << 32) | roi;
    }
    const int nkept = __syncthreads_count(kept[t]);
    sk[t] = k2;
    __syncthreads();
    cta_bitonic_sort(sk, SEL_N);
    if (t < DET_MAX) {
        float* o = dets + t * 6;
        float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
        if (t < nkept) {
            const unsigned roi = (unsigned)(sk[t] & 0xFFFFFFFFull);
            b = boxes[roi];
            o[4] = (float)(keys[roi] >> 42);
            o[5] = scores[roi];
        } else { o[4] = 0.f; o[5] = 0.f; }
        o[0] = b.x; o[1] = b.y; o[2] = b.z; o[3] = b.w;
        dboxes[t] = b;
    }
    if (t == 0) *count = nkept < DET_MAX ? nkept : DET_MAX;
}

// R-SIGMOID of each detection's own class: mask logits rows [det][y][x][dy][dx] x 128 -> masks [det][2y + dy][2x + dx]
__global__ void k_mask_select(const float* __restrict__ mlog, const float* __restrict__ dets, float* __restrict__ masks)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= DET_MAX * MASK * MASK) return;
    const int d = t / (MASK * MASK), Y = (t / MASK) % MASK, X = t % MASK;
    const int cls = (int)dets[d * 6 + 4];
    const size_t row = (((size_t)d * MPOOL + (Y >> 1)) * MPOOL + (X >> 1)) * 4 + (Y & 1) * 2 + (X & 1);
    masks[t] = 1.0f / (1.0f + det_expf(-mlog[row * MLOG_N + cls]));
}

// R-UNMOLD + the export rule, one thread: detections (window-normalised) -> exported boxes in image pixels, ids, class ids, rois
// einfo = {exported count, error (special assignment out of range)}; ebox = y1 x1 y2 x2 detection-row per exported detection
__global__ void k_unmold(const float* __restrict__ dets, float4 win, int W, int H, ExportParams ep, int* __restrict__ ebox, uint8_t* __restrict__ eid,
                         int* __restrict__ ecls, int* __restrict__ erois, int* __restrict__ einfo)
{
    int N = DET_MAX;
    for (int d = 0; d < DET_MAX; ++d)
        if (dets[d * 6 + 4] == 0.0f) { N = d; break; }
    const float wh = win.z - win.x, ww = win.w - win.y;
    int n = 0, err = 0;
    for (int d = 0; d < N; ++d) {
        const float* r = dets + d * 6;
        const float ny1 = (r[0] - win.x) / wh, nx1 = (r[1] - win.y) / ww, ny2 = (r[2] - win.x) / wh, nx2 = (r[3] - win.y) / ww;
        const int y1 = (int)rint((double)ny1 * (double)(H - 1) + 0.0), x1 = (int)rint((double)nx1 * (double)(W - 1) + 0.0);
        const int y2 = (int)rint((double)ny2 * (double)(H - 1) + 1.0), x2 = (int)rint((double)nx2 * (double)(W - 1) + 1.0);
        if ((y2 - y1) * (x2 - x1) <= 0) continue;
        const int cid = (int)r[4];
        uint8_t id = 0;
        const int e = id_export(cid, r[5], ep.min_score, ep.filter, ep.n_filter, ep.special, ep.n_special, n, &id);
        if (e < 0) { err = 1; break; }
        if (e == 0) continue;
        ebox[n * 5 + 0] = y1; ebox[n * 5 + 1] = x1; ebox[n * 5 + 2] = y2; ebox[n * 5 + 3] = x2; ebox[n * 5 + 4] = d;
        eid[n] = id;
        ecls[n] = cid;
        erois[n * 4 + 0] = y1; erois[n * 4 + 1] = x1; erois[n * 4 + 2] = y2; erois[n * 4 + 3] = x2;
        ++n;
    }
    einfo[0] = err ? 0 : n;
    einfo[1] = err;
}

// R-RESIZE value of a 28x28 mask resized to h x w at output pixel (r, c): fp64 bilinear with zero outside the grid, rounded to fp32
MF_D float resized_mask(const float* __restrict__ m, int h, int w, int r, int c)
{
    const double cy = ((double)r + 0.5) * (28.0 / (double)h) - 0.5, cx = ((double)c + 0.5) * (28.0 / (double)w) - 0.5;
    const double fy0 = floor(cy), fx0 = floor(cx);
    const int iy = (int)fy0, ix = (int)fx0;
    const double fy = cy - fy0, fx = cx - fx0;
    const bool y0 = iy >= 0 && iy < MASK, y1 = iy + 1 >= 0 && iy + 1 < MASK, x0 = ix >= 0 && ix < MASK, x1 = ix + 1 >= 0 && ix + 1 < MASK;
    const double v00 = y0 && x0 ? (double)m[iy * MASK + ix] : 0.0, v01 = y0 && x1 ? (double)m[iy * MASK + ix + 1] : 0.0;
    const double v10 = y1 && x0 ? (double)m[(iy + 1) * MASK + ix] : 0.0, v11 = y1 && x1 ? (double)m[(iy + 1) * MASK + ix + 1] : 0.0;
    const double top = (1.0 - fx) * v00 + fx * v01, bot = (1.0 - fx) * v10 + fx * v11;
    return (float)((1.0 - fy) * top + fy * bot);
}

// one thread per image pixel: the last exported detection whose box holds the pixel and whose resized mask is >= 0.5 there gives the id
__global__ void k_paste(const float* __restrict__ masks, const int* __restrict__ ebox, const uint8_t* __restrict__ eid, const int* __restrict__ einfo,
                        int W, int H, uint8_t* __restrict__ out)
{
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= W * H) return;
    const int y = p / W, x = p - (p / W) * W;
    uint8_t v = 0;
    for (int e = einfo[0] - 1; e >= 0; --e) {
        const int* b = ebox + e * 5;
        if (y < b[0] || y >= b[2] || x < b[1] || x >= b[3]) continue;
        if (resized_mask(masks + (size_t)b[4] * MASK * MASK, b[2] - b[0], b[3] - b[1], y - b[0], x - b[1]) >= 0.5f) { v = eid[e]; break; }
    }
    out[p] = v;
}

// hand-off to segmentation (FrameData::mask / classIDs, MaskRCNN.cpp:98-112): 16 id-image bytes per thread into the frame's mask, block 0
// also writes the header.  An export error left einfo = {0, 1} and an all-zero id image: the frame carries no masks.  A frame the caller
// gave a mask keeps it (the detector rank of a sharded run detects before it can know; one process never detects such a frame).
__global__ void k_frame_masks(const uint4* __restrict__ idimg, const int* __restrict__ einfo, const int* __restrict__ ecls, int n16,
                              uint4* __restrict__ mask, FrameHdr* __restrict__ hdr)
{
    if (hdr->maskGiven) return;
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < n16) mask[t] = idimg[t];
    if (blockIdx.x != 0) return;
    const int err = einfo[1], n = err ? 0 : einfo[0] + 1;
    for (int i = threadIdx.x; i < 256; i += blockDim.x) hdr->classIDs[i] = (i > 0 && i < n) ? ecls[i - 1] : 0;
    if (threadIdx.x == 0) { hdr->nMasks = n; hdr->detectError = err; }
}

}  // namespace mfb

using namespace mfb;

struct mf_detector {
    mf_rpn* rpn;
    mf_backbone* bb;
    cudaStream_t s;
    WeightStore w;
    int S = 0, imgW = 0, imgH = 0;
    float4 win = make_float4(0.f, 0.f, 1.f, 1.f);             // letter-box window of the current image, normalised (norm_boxes)
    ExportParams ep;
    DevBuf<__nv_bfloat16> fc1, fc2, mpool, col, mconv[4], dec;
    DevBuf<float> head, mlog, masks, dets, scores;
    DevBuf<float4> boxes, dboxes;
    DevBuf<unsigned long long> keys;
    DevBuf<int> count, ebox, ecls, erois, einfo;
    DevBuf<uint8_t> eid, idimg;                               // idimg: sized for the largest image so far
    mf_detector(mf_rpn* rpn, unsigned seed);                  // throws CudaError
};

// the image geometry: the letter-box window of a W x H image in the S x S input, normalised as norm_boxes does (float64 divide, float32)
static void set_image(mf_detector* h, int W, int H)
{
    if (W < 1 || H < 1 || W > 16384 || H > 16384)
        throw CudaError{"detector: image size " + std::to_string(W) + "x" + std::to_string(H) + " outside [1, 16384]"};
    if ((size_t)W * H > h->idimg.n) {
        if (cudaStreamSynchronize(h->s) != cudaSuccess) throw CudaError{"detector: id image free failed"};
        try {
            h->idimg.alloc((size_t)W * H);
        } catch (const CudaError& e) {
            throw CudaError{"detector: id image " + e.what};
        }
    }
    const MoldGeom g = cnn_mold_geometry(h->S, W, H);
    const double s1 = (double)(h->S - 1);
    h->win = make_float4((float)(g.offy / s1), (float)(g.offx / s1), (float)((g.offy + g.newH - 1) / s1), (float)((g.offx + g.newW - 1) / s1));
    h->imgW = W; h->imgH = H;
}

static void gemm(mf_detector* h, int layer, const void* A, void* out, int M, int relu, bool f32)
{
    const LayerGeom L = mrcnn_layer(MRCNN_DETECTOR, layer);
    launch_gemm_bf16(A, h->w.w(layer), h->w.b(layer), nullptr, out, M, L.rows, L.K, relu, h->s, nullptr, f32);
}

static void refine(mf_detector* h, const float* rois, const float* logits, int lstride, const float* deltas, int dstride, int n)
{
    const Enq q{h->s, nullptr};
    launch(q, nullptr, k_det_refine, (n + 127) / 128, 128, 0, (const float4*)rois, logits, lstride, deltas, dstride, n, h->win, h->keys.p, h->boxes.p,
           h->scores.p);
    launch(q, nullptr, k_det_select, 1, SEL_N, 0, h->keys.p, n, h->boxes.p, h->scores.p, h->dets.p, h->dboxes.p, h->count.p);
}

static void paste(mf_detector* h, const float* dets, const float* masks)
{
    const Enq q{h->s, nullptr};
    launch(q, nullptr, k_unmold, 1, 1, 0, dets, h->win, h->imgW, h->imgH, h->ep, h->ebox.p, h->eid.p, h->ecls.p, h->erois.p, h->einfo.p);
    launch(q, nullptr, k_paste, (h->imgW * h->imgH + 255) / 256, 256, 0, masks, h->ebox.p, h->eid.p, h->einfo.p, h->imgW, h->imgH, h->idimg.p);
}

mf_detector::mf_detector(mf_rpn* rpn_, unsigned seed) : rpn(rpn_), bb(rpn_backbone(rpn_)), s(backbone_stream(bb)), w(MRCNN_DETECTOR, seed, s)
{
    const LayerGeom fc1L = mrcnn_layer(MRCNN_DETECTOR, L_FC1), headL = mrcnn_layer(MRCNN_DETECTOR, L_HEAD), m1 = mrcnn_layer(MRCNN_DETECTOR, L_M1),
                    decL = mrcnn_layer(MRCNN_DETECTOR, L_DECONV), mlogL = mrcnn_layer(MRCNN_DETECTOR, L_MLOG);
    assert(mrcnn_num_layers(MRCNN_DETECTOR) == N_LAYERS && fc1L.rows == FC_N && fc1L.K == POOL * POOL * CH && headL.rows == HEAD_N &&
           m1.rows == CH && m1.K == MCONV_K && decL.rows == 4 * CH && mlogL.rows == MLOG_N);     // the shapes the buffers and kernels assume
    int d[3];
    backbone_level(bb, 4, d);
    S = d[0] * 4;
    imgW = imgH = S;                                          // the S x S image: its letter-box window is the whole input, `win`'s default
    memset(&ep, 0, sizeof ep);
    ep.min_score = 0.55;
    const size_t mrows = (size_t)DET_MAX * MPIX;
    fc1.alloc((size_t)DET_ROIS * FC_N); fc2.alloc((size_t)DET_ROIS * FC_N); head.alloc((size_t)DET_ROIS * HEAD_N); keys.alloc(DET_ROIS);
    boxes.alloc(DET_ROIS); scores.alloc(DET_ROIS); dets.alloc(DET_MAX * 6); dboxes.alloc(DET_MAX); count.alloc(1);
    mpool.alloc(mrows * CH); col.alloc(mrows * MCONV_K); dec.alloc(mrows * 4 * CH); mlog.alloc(mrows * 4 * MLOG_N);
    masks.alloc(DET_MAX * MASK * MASK); ebox.alloc(DET_MAX * 5); ecls.alloc(DET_MAX); erois.alloc(DET_MAX * 4); einfo.alloc(2); eid.alloc(DET_MAX);
    idimg.alloc((size_t)S * S);
    for (int i = 0; i < 4; ++i) mconv[i].alloc(mrows * CH);
    cudaCheck(cudaMemset(dets, 0, DET_MAX * 6 * 4), "cudaMemset");
    cudaCheck(cudaMemset(count, 0, 4), "cudaMemset");
    cudaCheck(cudaMemset(masks, 0, DET_MAX * MASK * MASK * 4), "cudaMemset");
    cudaCheck(cudaMemset(einfo, 0, 8), "cudaMemset");
}

namespace mfb {
cudaStream_t detector_stream(mf_detector* h) { return h->s; }

void detector_reserve_image(mf_detector* h, int W, int H) { set_image(h, W, H); }

void detector_frame_masks(mf_detector* h, uint8_t* mask, FrameHdr* hdr)
{
    const size_t P = (size_t)h->imgW * h->imgH;
    if (P % 16 || ((uintptr_t)mask & 15)) throw CudaError{"detector: the frame mask needs W x H % 16 == 0 and a 16-byte aligned buffer"};
    const int n16 = (int)(P / 16);
    launch(Enq{h->s, nullptr}, nullptr, k_frame_masks, (n16 + 255) / 256, 256, 0, (const uint4*)h->idimg.p, h->einfo.p, h->ecls.p, n16, (uint4*)mask,
           hdr);
}

void detector_run(mf_detector* h, int stages)
{
    if (stages & MF_DET_CLASSIFIER) {
        gemm(h, L_FC1, rpn_pooled(h->rpn), h->fc1, DET_ROIS, 1, false);
        gemm(h, L_FC2, h->fc1, h->fc2, DET_ROIS, 1, false);
        gemm(h, L_HEAD, h->fc2, h->head, DET_ROIS, 0, true);
    }
    if (stages & MF_DET_DETECTIONS) refine(h, rpn_rois(h->rpn), h->head, HEAD_N, h->head + NCLS, HEAD_N, DET_ROIS);
    if (stages & MF_DET_MASKS) {
        roi_align(h->bb, (const float*)h->dboxes.p, DET_MAX, MPOOL, h->mpool);
        const __nv_bfloat16* x = h->mpool;
        for (int i = 0; i < 4; ++i) {
            launch_im2col(x, DET_MAX, MPOOL, MPOOL, CH, MPOOL, MPOOL, 3, 1, 1, MCONV_K, h->col, h->s);
            gemm(h, L_M1 + i, h->col, h->mconv[i], DET_MAX * MPIX, 1, false);
            x = h->mconv[i];
        }
        gemm(h, L_DECONV, x, h->dec, DET_MAX * MPIX, 1, false);
        gemm(h, L_MLOG, h->dec, h->mlog, DET_MAX * MPIX * 4, 0, true);
        launch(Enq{h->s, nullptr}, nullptr, k_mask_select, (DET_MAX * MASK * MASK + 255) / 256, 256, 0, h->mlog.p, h->dets.p, h->masks.p);
    }
    if (stages & MF_DET_ID_IMAGE) paste(h, h->dets, h->masks);
}

void detector_detect(mf_detector* h, const void* d_rgba, int W, int H)
{
    set_image(h, W, H);
    backbone_mold(h->bb, d_rgba, W, H);
    backbone_forward(h->bb, backbone_input(h->bb));
    rpn_run(h->rpn, MF_RPN_CONV | MF_RPN_HEADS | MF_RPN_PROPOSALS | MF_RPN_ROI_ALIGN);
    detector_run(h, MF_DET_CLASSIFIER | MF_DET_DETECTIONS | MF_DET_MASKS | MF_DET_ID_IMAGE);
}
}  // namespace mfb

// ==========================================================================================
// C ABI (declared in include/maskfusion_b200.h)
// ==========================================================================================
extern "C" mf_detector* mf_detector_create(mf_rpn* rpn, unsigned seed)
{
    MF_TRY
    if (!rpn) { mf_set_error("detector: no region-proposal handle"); return nullptr; }
    return new mf_detector(rpn, seed);
    MF_CATCH_AS(nullptr, "detector: ")
}

extern "C" void mf_detector_destroy(mf_detector* h) { delete h; }

extern "C" int mf_detector_run(mf_detector* h, int stages)
{
    MF_TRY
    if (!h) throw CudaError{"detector: null handle"};
    detector_run(h, stages);
    return 0;
    MF_CATCH(-1)
}

extern "C" int mf_detector_forward(mf_detector* h, int image_w, int image_h)
{
    MF_TRY
    if (!h) throw CudaError{"detector: null handle"};
    set_image(h, image_w, image_h);
    detector_run(h, MF_DET_CLASSIFIER | MF_DET_DETECTIONS | MF_DET_MASKS | MF_DET_ID_IMAGE);
    return 0;
    MF_CATCH(-1)
}

extern "C" int mf_detector_detect(mf_detector* h, const void* d_rgba, int W, int H)
{
    MF_TRY
    if (!h) throw CudaError{"detector: null handle"};
    if (!d_rgba || ((uintptr_t)d_rgba & 3)) throw CudaError{"detector: the image needs a 4-byte aligned device pointer"};
    detector_detect(h, d_rgba, W, H);
    return 0;
    MF_CATCH(-1)
}

extern "C" int mf_detector_set_export(mf_detector* h, double min_score, const int32_t* class_filter, int n_filter, const int32_t* special_assignments,
                                      int n_special)
{
    MF_TRY
    if (!h) throw CudaError{"detector: null handle"};
    if (n_filter < 0 || n_special < 0 || n_filter > EXPORT_CAP || n_special > EXPORT_CAP || (n_filter && !class_filter) || (n_special && !special_assignments))
        throw CudaError{"detector_set_export: lists of 0.." + std::to_string(EXPORT_CAP) + " entries"};
    ExportParams ep;
    memset(&ep, 0, sizeof ep);
    ep.min_score = min_score; ep.n_filter = n_filter; ep.n_special = n_special;
    for (int i = 0; i < n_filter; ++i) ep.filter[i] = class_filter[i];
    for (int i = 0; i < n_special; ++i) ep.special[i] = special_assignments[i];
    h->ep = ep;
    return 0;
    MF_CATCH(-1)
}

extern "C" int mf_detector_refine(mf_detector* h, const float* d_rois, const float* d_logits, const float* d_deltas, int n)
{
    MF_TRY
    if (!h) throw CudaError{"detector: null handle"};
    if (n < 1 || n > DET_ROIS) throw CudaError{"detector_refine: n = " + std::to_string(n) + " outside [1, 1000]"};
    if (!d_rois || !d_logits || !d_deltas || ((uintptr_t)d_rois & 15) || ((uintptr_t)d_logits & 3) || ((uintptr_t)d_deltas & 3))
        throw CudaError{"detector_refine: rois need a 16-byte, logits and deltas a 4-byte aligned device pointer"};
    refine(h, d_rois, d_logits, NCLS, d_deltas, 4 * NCLS, n);
    return 0;
    MF_CATCH(-1)
}

extern "C" int mf_detector_paste(mf_detector* h, const float* d_detections, const float* d_masks, int W, int H)
{
    MF_TRY
    if (!h) throw CudaError{"detector: null handle"};
    if (!d_detections || !d_masks || ((uintptr_t)d_detections & 3) || ((uintptr_t)d_masks & 3))
        throw CudaError{"detector_paste: detections and masks need 4-byte aligned device pointers"};
    set_image(h, W, H);
    paste(h, d_detections, d_masks);
    return 0;
    MF_CATCH(-1)
}

extern "C" int mf_detector_num_layers(mf_detector* h) { return h ? N_LAYERS : -1; }

extern "C" int mf_detector_layer(mf_detector* h, int i, int* out6)
{
    MF_TRY
    if (!h || i < 0 || i >= N_LAYERS || !out6) throw CudaError{"detector: bad layer index"};
    const LayerGeom L = mrcnn_layer(MRCNN_DETECTOR, i);
    out6[0] = L.cin; out6[1] = L.rows; out6[2] = L.k; out6[3] = L.stride; out6[4] = L.pad; out6[5] = L.K;
    return 0;
    MF_CATCH(-1)
}

extern "C" int mf_detector_get_weights(mf_detector* h, int i, float* w, float* bias)
{
    MF_TRY
    if (!h) throw CudaError{"detector: bad layer index"};
    h->w.get(i, w, bias);
    return 0;
    MF_CATCH(-1)
}

// pretrained weights (mf_weights.cu): read, checked and folded on the host first; the copy is ordered on the stream and complete on return
extern "C" int mf_detector_load_weights(mf_detector* h, const char* path)
{
    MF_TRY
    if (!h) throw CudaError{"detector: null handle"};
    h->w.load(path, h->s);
    return 0;
    MF_CATCH(-1)
}

extern "C" int mf_detector_get_fc(mf_detector* h, void* fc1_bf16, void* fc2_bf16)
{
    MF_TRY
    if (!h) throw CudaError{"detector: null handle"};
    cnn_read_back(h->s, fc1_bf16, h->fc1, (size_t)DET_ROIS * FC_N * 2);
    cnn_read_back(h->s, fc2_bf16, h->fc2, (size_t)DET_ROIS * FC_N * 2);
    return 0;
    MF_CATCH(-1)
}

extern "C" int mf_detector_get_head_outputs(mf_detector* h, float* logits, float* deltas)
{
    MF_TRY
    if (!h) throw CudaError{"detector: null handle"};
    cnn_read_back(h->s, logits, h->head, NCLS * 4, DET_ROIS, HEAD_N * 4);
    cnn_read_back(h->s, deltas, h->head.p + NCLS, NCLS * 16, DET_ROIS, HEAD_N * 4);
    return 0;
    MF_CATCH(-1)
}

extern "C" int mf_detector_get_mask_layer(mf_detector* h, int i, void* host)
{
    MF_TRY
    if (!h) throw CudaError{"detector: null handle"};
    const size_t px = (size_t)DET_MAX * MPIX;
    switch (i) {
    case 0: cnn_read_back(h->s, host, h->mpool, px * CH * 2); break;
    case 1: case 2: case 3: case 4: cnn_read_back(h->s, host, h->mconv[i - 1], px * CH * 2); break;
    case 5: cnn_read_back(h->s, host, h->dec, px * 4 * CH * 2); break;
    case 6: cnn_read_back(h->s, host, h->mlog, NCLS * 4, px * 4, MLOG_N * 4); break;
    default: throw CudaError{"detector: mask layer must be 0..6"};
    }
    return 0;
    MF_CATCH(-1)
}

extern "C" int mf_detector_get_detections(mf_detector* h, float* detections)
{
    MF_TRY
    if (!h) throw CudaError{"detector: null handle"};
    int n = 0;
    cnn_read_back(h->s, detections, h->dets, DET_MAX * 6 * 4);
    cnn_read_back(h->s, &n, h->count, 4);
    return n;
    MF_CATCH(-1)
}

extern "C" int mf_detector_get_masks(mf_detector* h, float* masks)
{
    MF_TRY
    if (!h) throw CudaError{"detector: null handle"};
    cnn_read_back(h->s, masks, h->masks, DET_MAX * MASK * MASK * 4);
    return 0;
    MF_CATCH(-1)
}

extern "C" int mf_detector_get_id_image(mf_detector* h, uint8_t* id_image, int32_t* class_ids, int32_t* rois)
{
    MF_TRY
    if (!h) throw CudaError{"detector: null handle"};
    int info[2];
    cnn_read_back(h->s, info, h->einfo, 8);
    if (info[1]) throw CudaError{"generate_id_image: special_assignments[class_id] out of range"};
    cnn_read_back(h->s, id_image, h->idimg, (size_t)h->imgW * h->imgH);
    cnn_read_back(h->s, class_ids, h->ecls, (size_t)info[0] * 4);
    cnn_read_back(h->s, rois, h->erois, (size_t)info[0] * 16);
    return info[0];
    MF_CATCH(-1)
}

extern "C" int mf_detector_image_size(mf_detector* h, int* w, int* hgt)
{
    MF_TRY
    if (!h) throw CudaError{"detector: null handle"};
    *w = h->imgW; *hgt = h->imgH;
    return 0;
    MF_CATCH(-1)
}
