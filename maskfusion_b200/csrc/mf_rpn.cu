// mf_rpn.cu -- Mask R-CNN region-proposal stage on the backbone's P2..P6 (sm_90a): RPN head, proposal layer, pyramid ROI Align.
//
// The network is matterport mrcnn's inference graph with the COCO InferenceConfig defaults, written from upstream memory (the source is not
// vendored; DESIGN §3c, rules R-TOPK / R-NMS / R-ROILEVEL in §4):
//   rpn_graph        shared 3x3 256->512 conv + ReLU on every level, 1x1 512->6 class logits (channel a*2+c), 1x1 512->12 box deltas
//                    (channel a*4+k, k = dy dx log(dh) log(dw)), 3 anchors per feature pixel
//   ProposalLayer    softmax score, deltas * RPN_BBOX_STD_DEV, top min(6000, A) by score, apply_box_deltas_graph, clip to [0,0,1,1],
//                    greedy NMS at IoU 0.7 up to 1000 boxes, zero padding to 1000
//   PyramidROIAlign  level from the box area, tf.image.crop_and_resize (bilinear) on P2..P5 -> [n][P][P][256] bf16 (NHWC per ROI)
// The 3x3 conv runs through the backbone's conv path (cnn_conv: implicit wgmma GEMM, or im2col + GEMM where its geometry guard refuses the
// shape); the two 1x1 heads are ONE wgmma GEMM over the concatenated conv outputs of all levels, 18 weight rows zero-padded to 64, with the
// fp32 epilogue.  Everything after the GEMMs is IEEE fp32 in a fixed operation order (this file is compiled -fmad=false), so proposals
// and pooled features are reproducible bit for bit by the numpy restatement in tests/rpn_ref.py.
//
// Proposal layer: a sequence of launches on one stream, no inter-CTA waits.
//   k_rpn_keys      key = ~ord(score) << 32 | anchor index: ascending key order is R-TOPK order; resets the selection state
//   k_sel_hist/pick radix select of the k-th smallest key, 8 bits per pass: 4 passes over the score bits, then the used anchor-index bits
//   k_sel_compact   the k keys <= the k-th one (unordered: slots from an atomic counter)
//   k_sort_decode   one CTA: bitonic sort of the k keys in shared memory, then apply_box_deltas + clip in R-TOPK order
//   k_nms_mask      IoU > 0.7 bitmask: candidate i x 64-candidate words (upper triangle only)
//   k_nms_scan      one warp: the greedy scan over the bitmask, stop at 1000 kept, zero padding
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

constexpr int RPN_PRE_NMS = 6000, RPN_POST_NMS = 1000, RPN_POOL = 7, RPN_CH = 256, RPN_MID = 512, RPN_HEAD_N = 64;
constexpr int NMS_WORDS = (RPN_PRE_NMS + 63) / 64;          // 94 words of 64 candidates
constexpr int SORT_CAP = 8192;                              // bitonic sort size >= RPN_PRE_NMS, 64 KB of keys in shared memory
constexpr float RPN_NMS_THRESHOLD = 0.7f;

struct SelState { unsigned long long prefix, mask; unsigned krem, nsel; unsigned hist[256]; };

// softmax over the two logits (Keras: exp(x - max) / sum) -> foreground score -> R-TOPK key; block 0 resets the selection state
__global__ void k_rpn_keys(const float2* __restrict__ logits, int n, int k, unsigned long long* __restrict__ keys, SelState* st)
{
    if (blockIdx.x == 0) {
        for (int t = threadIdx.x; t < 256; t += blockDim.x) st->hist[t] = 0;
        if (threadIdx.x == 0) { st->prefix = 0; st->mask = 0; st->krem = (unsigned)k; st->nsel = 0; }
    }
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float2 l = logits[i];
        const float m = l.y > l.x ? l.y : l.x;
        const float e0 = det_expf(l.x - m), e1 = det_expf(l.y - m);
        const float score = e1 / (e0 + e1);
        keys[i] = ((unsigned long long)(~score_ord(score)) << 32) | (unsigned)i;
    }
}

// histogram of the 8-bit digit at `shift` over the keys that match the prefix selected so far
__global__ void k_sel_hist(const unsigned long long* __restrict__ keys, int n, SelState* st, int shift)
{
    __shared__ unsigned h[256];
    for (int t = threadIdx.x; t < 256; t += blockDim.x) h[t] = 0;
    __syncthreads();
    const unsigned long long mask = st->mask, prefix = st->prefix;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const unsigned long long key = keys[i];
        if ((key & mask) == prefix) atomicAdd(&h[(key >> shift) & 255], 1u);
    }
    __syncthreads();
    for (int t = threadIdx.x; t < 256; t += blockDim.x)
        if (h[t]) atomicAdd(&st->hist[t], h[t]);
}

// the digit bin that holds the krem-th smallest matching key joins the prefix; the histogram is cleared for the next pass
__global__ void k_sel_pick(SelState* st, int shift)
{
    __shared__ unsigned h[256];
    h[threadIdx.x] = st->hist[threadIdx.x];
    st->hist[threadIdx.x] = 0;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned cum = 0;
        for (int d = 0; d < 256; ++d) {
            if (cum + h[d] >= st->krem) {
                st->prefix |= (unsigned long long)d << shift;
                st->mask |= 0xFFull << shift;
                st->krem -= cum;
                break;
            }
            cum += h[d];
        }
    }
}

// keys are unique (the anchor index is in the low half): exactly k of them are <= the k-th smallest
__global__ void k_sel_compact(const unsigned long long* __restrict__ keys, int n, SelState* st, unsigned long long* __restrict__ sel)
{
    const unsigned long long kth = st->prefix;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const unsigned long long key = keys[i];
        if (key <= kth) sel[atomicAdd(&st->nsel, 1u)] = key;
    }
}

// one CTA: bitonic sort of the k selected keys (padded with ~0 to a power of two), then the boxes in R-TOPK order
__global__ void __launch_bounds__(1024) k_sort_decode(const unsigned long long* __restrict__ sel, int k, const float4* __restrict__ deltas,
                                                      const float4* __restrict__ anchors, float4* __restrict__ boxes)
{
    extern __shared__ unsigned long long sk[];
    int P = 1;
    while (P < k) P <<= 1;
    for (int i = threadIdx.x; i < P; i += blockDim.x) sk[i] = i < k ? sel[i] : ~0ull;
    __syncthreads();
    cta_bitonic_sort(sk, P);
    for (int i = threadIdx.x; i < k; i += blockDim.x) {
        const unsigned idx = (unsigned)(sk[i] & 0xFFFFFFFFull);
        boxes[i] = decode_box(anchors[idx], deltas[idx], make_float4(0.f, 0.f, 1.f, 1.f));
    }
}

// bit j of word (i, c) set <=> candidate 64c + j comes after i and IoU(i, 64c + j) > 0.7; words left of the diagonal are not written
__global__ void __launch_bounds__(64) k_nms_mask(const float4* __restrict__ boxes, int k, int words, unsigned long long* __restrict__ mask)
{
    const int row = blockIdx.y, col = blockIdx.x;
    if (col < row) return;
    const int rowSize = min(k - row * 64, 64), colSize = min(k - col * 64, 64);
    __shared__ float4 cb[64];
    if ((int)threadIdx.x < colSize) cb[threadIdx.x] = boxes[col * 64 + threadIdx.x];
    __syncthreads();
    if ((int)threadIdx.x >= rowSize) return;
    const int i = row * 64 + threadIdx.x;
    const float4 bi = boxes[i];
    unsigned long long bits = 0;
    for (int j = row == col ? threadIdx.x + 1 : 0; j < colSize; ++j)
        if (iou_tf(bi, cb[j]) > RPN_NMS_THRESHOLD) bits |= 1ull << j;
    mask[(size_t)i * words + col] = bits;
}

// one warp, greedy in R-TOPK order; lane l holds the suppression words l, l + 32, l + 64
__global__ void __launch_bounds__(32) k_nms_scan(const float4* __restrict__ boxes, const unsigned long long* __restrict__ mask, int k, int words,
                                                 float4* __restrict__ rois, int* __restrict__ count)
{
    const int lane = threadIdx.x;
    unsigned long long r0 = 0, r1 = 0, r2 = 0;
    int kept = 0;
    for (int i = 0; i < k && kept < RPN_POST_NMS; ++i) {
        const int w = i >> 6, slot = w >> 5;
        const unsigned long long mine = slot == 0 ? r0 : (slot == 1 ? r1 : r2);
        const unsigned long long v = __shfl_sync(0xFFFFFFFFu, mine, w & 31);
        if ((v >> (i & 63)) & 1ull) continue;
        if (lane == 0) rois[kept] = boxes[i];
        ++kept;
        const unsigned long long* row = mask + (size_t)i * words;
        if (lane >= w && lane < words) r0 |= row[lane];
        if (lane + 32 >= w && lane + 32 < words) r1 |= row[lane + 32];
        if (lane + 64 >= w && lane + 64 < words) r2 |= row[lane + 64];
    }
    for (int j = kept + lane; j < RPN_POST_NMS; j += 32) rois[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (lane == 0) *count = kept;
}

// head GEMM rows [pixel][64] (0..5 logits, 6..17 deltas) -> logits [A][2], deltas [A][4] with anchor = 3 * pixel + a
__global__ void k_rpn_split(const float* __restrict__ head, int pixels, float* __restrict__ logits, float* __restrict__ deltas)
{
    const int total = pixels * 18;
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < total; t += gridDim.x * blockDim.x) {
        const int p = t / 18, c = t - p * 18;
        const float v = head[(size_t)p * RPN_HEAD_N + c];
        if (c < 6) logits[(size_t)p * 6 + c] = v;
        else deltas[(size_t)p * 12 + c - 6] = v;
    }
}

// ---- pyramid ROI Align (tf.image.crop_and_resize, bilinear, extrapolation value 0) ----
struct RoiLevels { const __nv_bfloat16* P[4]; int H[4], W[4]; };

// R-ROILEVEL: t = h*w * fp32(S^2 / 224^2) against the exact boundaries of 4 + round(log2(sqrt(h*w) * S / 224)); NaN / degenerate -> 2
MF_D int roi_level(float4 b, float areaScale)
{
    const float t = ((b.z - b.x) * (b.w - b.y)) * areaScale;
    return 2 + (t >= 0.125f) + (t >= 0.5f) + (t >= 2.0f);
}

// block (roi, output row), thread = channel pair; out [n][P][P][256] bf16, each value rounded once from the fp32 interpolation
__global__ void __launch_bounds__(128) k_roi_align(const float4* __restrict__ boxes, int pool, RoiLevels lv, float areaScale,
                                                   __nv_bfloat16* __restrict__ out)
{
    const int roi = blockIdx.x, iy = blockIdx.y, c = 2 * threadIdx.x;
    const float4 b = boxes[roi];
    const int li = roi_level(b, areaScale) - 2;                     // selects, not an indexed load: the parameter struct stays in registers
    const __nv_bfloat16* f = li == 0 ? lv.P[0] : li == 1 ? lv.P[1] : li == 2 ? lv.P[2] : lv.P[3];
    const int H = li == 0 ? lv.H[0] : li == 1 ? lv.H[1] : li == 2 ? lv.H[2] : lv.H[3];
    const int W = li == 0 ? lv.W[0] : li == 1 ? lv.W[1] : li == 2 ? lv.W[2] : lv.W[3];
    const float hs = ((b.z - b.x) * (float)(H - 1)) / (float)(pool - 1);
    const float ws = ((b.w - b.y) * (float)(W - 1)) / (float)(pool - 1);
    const float in_y = b.x * (float)(H - 1) + (float)iy * hs;
    __nv_bfloat162* o = reinterpret_cast<__nv_bfloat162*>(out + (((size_t)roi * pool + iy) * pool) * RPN_CH + c);
    const __nv_bfloat162 zero = __floats2bfloat162_rn(0.f, 0.f);
    if (!(in_y >= 0.0f && in_y <= (float)(H - 1))) {               // outside the map (or NaN): the whole row is the extrapolation value
        for (int ix = 0; ix < pool; ++ix) o[ix * (RPN_CH / 2)] = zero;
        return;
    }
    const int ty = (int)floorf(in_y), by = (int)ceilf(in_y);
    const float yl = in_y - (float)ty;
    for (int ix = 0; ix < pool; ++ix) {
        const float in_x = b.y * (float)(W - 1) + (float)ix * ws;
        if (!(in_x >= 0.0f && in_x <= (float)(W - 1))) { o[ix * (RPN_CH / 2)] = zero; continue; }
        const int lx = (int)floorf(in_x), rx = (int)ceilf(in_x);
        const float xl = in_x - (float)lx;
        const float2 tl = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(f + ((size_t)ty * W + lx) * RPN_CH + c));
        const float2 tr = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(f + ((size_t)ty * W + rx) * RPN_CH + c));
        const float2 bl = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(f + ((size_t)by * W + lx) * RPN_CH + c));
        const float2 br = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(f + ((size_t)by * W + rx) * RPN_CH + c));
        const float t0 = tl.x + (tr.x - tl.x) * xl, t1 = tl.y + (tr.y - tl.y) * xl;
        const float b0 = bl.x + (br.x - bl.x) * xl, b1 = bl.y + (br.y - bl.y) * xl;
        o[ix * (RPN_CH / 2)] = __floats2bfloat162_rn(t0 + (b0 - t0) * yl, t1 + (b1 - t1) * yl);
    }
}

}  // namespace mfb

using namespace mfb;

struct mf_rpn {
    mf_backbone* bb;
    cudaStream_t s;
    WeightStore w;                                           // conv [512 x 2304], heads [64 x 512] (rows >= 18 zero)
    int S = 0, A = 0, pixels = 0;
    int lh[5] = {}, pixOff[6] = {};                          // P2..P6 side length, first pixel of each level in the concatenation
    DevBuf<__nv_bfloat16> col, conv, pooled;
    DevBuf<float> head, logits, deltas, anchors, rois;
    DevBuf<unsigned long long> keys, sel, mask;
    DevBuf<SelState> st;
    DevBuf<float4> boxes;
    DevBuf<int> count;
    mf_rpn(mf_backbone* bb, unsigned seed);                  // throws CudaError
};

static RoiLevels roi_levels(mf_backbone* bb)
{
    RoiLevels lv;
    for (int i = 0; i < 4; ++i) {
        int d[3];
        lv.P[i] = (const __nv_bfloat16*)backbone_level(bb, 4 + i, d);
        lv.H[i] = d[0]; lv.W[i] = d[1];
    }
    return lv;
}

void mfb::roi_align(mf_backbone* bb, const float* boxes, int n, int pool, void* out)
{
    if (n == 0) return;
    int d[3];
    backbone_level(bb, 4, d);
    const int S = d[0] * 4;
    const float areaScale = (float)((double)S * (double)S / (224.0 * 224.0));
    launch(Enq{backbone_stream(bb), nullptr}, nullptr, k_roi_align, dim3(n, pool), RPN_CH / 2, 0, (const float4*)boxes, pool, roi_levels(bb), areaScale,
           (__nv_bfloat16*)out);
}

// the proposal layer on logits [n][2], deltas [n][4], anchors [n][4] (device) -> h->rois [1000][4], h->count
static void propose(mf_rpn* h, const float* logits, const float* deltas, const float* anchors, int n)
{
    const Enq q{h->s, nullptr};
    const int k = n < RPN_PRE_NMS ? n : RPN_PRE_NMS;
    const int grid = (n + 255) / 256, histGrid = std::min((n + 2047) / 2048, 2 * num_sms());
    launch(q, nullptr, k_rpn_keys, grid, 256, 0, (const float2*)logits, n, k, h->keys.p, h->st.p);
    int shifts[8], np = 0;
    for (int sh = 56; sh >= 32; sh -= 8) shifts[np++] = sh;
    int idxBits = 0;
    while (idxBits < 32 && ((n - 1) >> idxBits)) ++idxBits;                  // anchor-index bits that vary
    for (int sh = 24; sh >= 0; sh -= 8)
        if (sh < idxBits) shifts[np++] = sh;
    for (int p = 0; p < np; ++p) {
        launch(q, nullptr, k_sel_hist, histGrid, 256, 0, h->keys.p, n, h->st.p, shifts[p]);
        launch(q, nullptr, k_sel_pick, 1, 256, 0, h->st.p, shifts[p]);
    }
    launch(q, nullptr, k_sel_compact, grid, 256, 0, h->keys.p, n, h->st.p, h->sel.p);
    launch(q, nullptr, k_sort_decode, 1, 1024, SORT_CAP * sizeof(unsigned long long), h->sel.p, k, (const float4*)deltas, (const float4*)anchors,
           h->boxes.p);
    const int words = (k + 63) / 64;
    launch(q, nullptr, k_nms_mask, dim3(words, words), 64, 0, h->boxes.p, k, words, h->mask.p);
    launch(q, nullptr, k_nms_scan, 1, 32, 0, h->boxes.p, h->mask.p, k, words, (float4*)h->rois.p, h->count.p);
}

void mfb::rpn_run(mf_rpn* h, int stages)
{
    const cudaStream_t s = h->s;
    if (stages & MF_RPN_CONV)
        for (int l = 0; l < 5; ++l) {
            int d[3];
            const void* in = backbone_level(h->bb, 4 + l, d);
            cnn_conv(in, d[0], d[1], RPN_CH, RPN_MID, 3, 1, 1, h->w.w(0), h->w.b(0), h->col, h->conv.p + (size_t)h->pixOff[l] * RPN_MID, 1, s);
        }
    if (stages & MF_RPN_HEADS) {
        launch_gemm_bf16(h->conv, h->w.w(1), h->w.b(1), nullptr, h->head, h->pixels, RPN_HEAD_N, RPN_MID, 0, s, nullptr, true);
        launch(Enq{s, nullptr}, nullptr, k_rpn_split, std::min((h->pixels * 18 + 255) / 256, 8 * num_sms()), 256, 0, h->head.p, h->pixels, h->logits.p,
               h->deltas.p);
    }
    if (stages & MF_RPN_PROPOSALS) propose(h, h->logits, h->deltas, h->anchors, h->A);
    if (stages & MF_RPN_ROI_ALIGN) roi_align(h->bb, h->rois, RPN_POST_NMS, RPN_POOL, h->pooled);
}

// ==========================================================================================
// C ABI (declared in include/maskfusion_b200.h)
// ==========================================================================================
mf_rpn::mf_rpn(mf_backbone* bb_, unsigned seed) : bb(bb_), s(backbone_stream(bb_)), w(MRCNN_RPN, seed, s)
{
    const LayerGeom c = mrcnn_layer(MRCNN_RPN, 0), hd = mrcnn_layer(MRCNN_RPN, 1);
    assert(c.cin == RPN_CH && c.rows == RPN_MID && hd.K == RPN_MID && hd.rows == RPN_HEAD_N);     // the shapes the kernels are compiled for
    int d[3];
    backbone_level(bb, 4, d);
    S = d[0] * 4;
    for (int l = 0; l < 5; ++l) {
        lh[l] = S >> (l + 2);
        pixOff[l + 1] = pixOff[l] + lh[l] * lh[l];
    }
    pixels = pixOff[5];
    A = 3 * pixels;
    // anchors: generate_pyramid_anchors + norm_boxes in double, rounded once to float; order (level, y, x, ratio)
    std::vector<float> anc((size_t)A * 4);
    const double ratios[3] = {0.5, 1.0, 2.0}, S1 = (double)(S - 1);
    size_t a = 0;
    for (int l = 0; l < 5; ++l) {
        const double scale = 32.0 * (1 << l), stride = 4.0 * (1 << l);
        for (int y = 0; y < lh[l]; ++y)
            for (int x = 0; x < lh[l]; ++x)
                for (int r = 0; r < 3; ++r, ++a) {
                    const double bh = scale / sqrt(ratios[r]), bw = scale * sqrt(ratios[r]), cy = y * stride, cx = x * stride;
                    anc[a * 4 + 0] = (float)((cy - 0.5 * bh) / S1);
                    anc[a * 4 + 1] = (float)((cx - 0.5 * bw) / S1);
                    anc[a * 4 + 2] = (float)((cy + 0.5 * bh - 1.0) / S1);
                    anc[a * 4 + 3] = (float)((cx + 0.5 * bw - 1.0) / S1);
                }
    }
    // im2col scratch only for the levels whose shape the implicit 3x3 path refuses
    size_t colElems = 0;
    for (int l = 0; l < 5; ++l)
        if (!cnn_conv_implicit(3, 1, 1, RPN_CH, lh[l], lh[l])) colElems = std::max(colElems, (size_t)lh[l] * lh[l] * c.K);
    col.alloc(colElems);
    conv.alloc((size_t)pixels * RPN_MID); head.alloc((size_t)pixels * RPN_HEAD_N);
    logits.alloc((size_t)A * 2); deltas.alloc((size_t)A * 4); anchors.alloc((size_t)A * 4); keys.alloc(A);
    sel.alloc(RPN_PRE_NMS); mask.alloc((size_t)RPN_PRE_NMS * NMS_WORDS); st.alloc(1); boxes.alloc(RPN_PRE_NMS);
    rois.alloc(RPN_POST_NMS * 4); count.alloc(1); pooled.alloc((size_t)RPN_POST_NMS * RPN_POOL * RPN_POOL * RPN_CH);
    cudaCheck(cudaMemcpy(anchors, anc.data(), anc.size() * 4, cudaMemcpyHostToDevice), "anchor upload");
    cudaCheck(cudaMemset(rois, 0, RPN_POST_NMS * 16), "cudaMemset");
    cudaCheck(cudaMemset(count, 0, 4), "cudaMemset");
    cudaCheck(cudaFuncSetAttribute(k_sort_decode, cudaFuncAttributeMaxDynamicSharedMemorySize, SORT_CAP * (int)sizeof(unsigned long long)),
              "cudaFuncSetAttribute");
}

extern "C" mf_rpn* mf_rpn_create(mf_backbone* bb, unsigned seed)
{
    MF_TRY
    if (!bb) { mf_set_error("rpn: no backbone"); return nullptr; }
    return new mf_rpn(bb, seed);
    MF_CATCH_AS(nullptr, "rpn: ")
}

extern "C" void mf_rpn_destroy(mf_rpn* h) { delete h; }

extern "C" int mf_rpn_run(mf_rpn* h, int stages)
{
    MF_TRY
    if (!h) throw CudaError{"rpn: null handle"};
    rpn_run(h, stages);
    return 0;
    MF_CATCH(-1)
}

extern "C" int mf_rpn_forward(mf_rpn* h)
{
    MF_TRY
    if (!h) throw CudaError{"rpn: null handle"};
    rpn_run(h, MF_RPN_CONV | MF_RPN_HEADS | MF_RPN_PROPOSALS | MF_RPN_ROI_ALIGN);
    return 0;
    MF_CATCH(-1)
}

extern "C" int mf_rpn_propose(mf_rpn* h, const float* d_logits, const float* d_deltas, const float* d_anchors, int n_anchors)
{
    MF_TRY
    if (!h) throw CudaError{"rpn: null handle"};
    if (n_anchors < 1 || n_anchors > h->A)
        throw CudaError{"rpn_propose: n_anchors = " + std::to_string(n_anchors) + " outside [1, " + std::to_string(h->A) + "]"};
    if (!d_logits || !d_deltas || !d_anchors || ((uintptr_t)d_logits & 7) || ((uintptr_t)d_deltas & 15) || ((uintptr_t)d_anchors & 15))
        throw CudaError{"rpn_propose: logits need 8-byte, deltas and anchors 16-byte aligned device pointers"};
    propose(h, d_logits, d_deltas, d_anchors, n_anchors);
    return 0;
    MF_CATCH(-1)
}

extern "C" int mf_roi_align_bf16(mf_backbone* bb, const float* d_boxes, int n, int pool, void* d_out)
{
    MF_TRY
    if (!bb) throw CudaError{"roi_align: no backbone"};
    if (n < 0 || pool < 2 || pool > 64) throw CudaError{"roi_align: need n >= 0 and 2 <= pool <= 64"};
    if (n > 0 && (!d_boxes || !d_out || ((uintptr_t)d_boxes & 15) || ((uintptr_t)d_out & 3)))
        throw CudaError{"roi_align: boxes need a 16-byte, out a 4-byte aligned device pointer"};
    roi_align(bb, d_boxes, n, pool, d_out);
    return 0;
    MF_CATCH(-1)
}

extern "C" int mf_rpn_num_anchors(mf_rpn* h) { return h ? h->A : -1; }

extern "C" int mf_rpn_get_weights(mf_rpn* h, float* conv_w, float* conv_b, float* head_w, float* head_b)
{
    MF_TRY
    if (!h) throw CudaError{"rpn: null handle"};
    h->w.get(0, conv_w, conv_b);
    h->w.get(1, head_w, head_b, 18);                         // head rows 0..5 logits, 6..17 deltas
    return 0;
    MF_CATCH(-1)
}

// pretrained weights (mf_weights.cu): read, checked and folded on the host first; the copy is ordered on the stream and complete on return
extern "C" int mf_rpn_load_weights(mf_rpn* h, const char* path)
{
    MF_TRY
    if (!h) throw CudaError{"rpn: null handle"};
    h->w.load(path, h->s);
    return 0;
    MF_CATCH(-1)
}

extern "C" int mf_rpn_get_anchors(mf_rpn* h, float* anchors)
{
    MF_TRY
    if (!h) throw CudaError{"rpn: null handle"};
    cnn_read_back(h->s, anchors, h->anchors, (size_t)h->A * 16);
    return 0;
    MF_CATCH(-1)
}

extern "C" int mf_rpn_get_head_outputs(mf_rpn* h, float* logits, float* deltas)
{
    MF_TRY
    if (!h) throw CudaError{"rpn: null handle"};
    cnn_read_back(h->s, logits, h->logits, (size_t)h->A * 8);
    cnn_read_back(h->s, deltas, h->deltas, (size_t)h->A * 16);
    return 0;
    MF_CATCH(-1)
}

extern "C" int mf_rpn_download_conv(mf_rpn* h, int level, void* host_bf16)
{
    MF_TRY
    if (!h) throw CudaError{"rpn: null handle"};
    if (level < 0 || level > 4) throw CudaError{"rpn: level must be 0..4 (P2..P6)"};
    cnn_read_back(h->s, host_bf16, h->conv.p + (size_t)h->pixOff[level] * RPN_MID, (size_t)h->lh[level] * h->lh[level] * RPN_MID * 2);
    return 0;
    MF_CATCH(-1)
}

extern "C" int mf_rpn_get_proposals(mf_rpn* h, float* rois)
{
    MF_TRY
    if (!h) throw CudaError{"rpn: null handle"};
    int n = 0;
    cnn_read_back(h->s, rois, h->rois, RPN_POST_NMS * 16);
    cnn_read_back(h->s, &n, h->count, 4);
    return n;
    MF_CATCH(-1)
}

extern "C" int mf_rpn_get_pooled(mf_rpn* h, void* host_bf16)
{
    MF_TRY
    if (!h) throw CudaError{"rpn: null handle"};
    cnn_read_back(h->s, host_bf16, h->pooled, (size_t)RPN_POST_NMS * RPN_POOL * RPN_POOL * RPN_CH * 2);
    return 0;
    MF_CATCH(-1)
}

// ---- what the detection heads (mf_heads.cu) read of the handle ----
mf_backbone* mfb::rpn_backbone(mf_rpn* h) { return h->bb; }
const float* mfb::rpn_rois(mf_rpn* h) { return h->rois; }
const void* mfb::rpn_pooled(mf_rpn* h) { return h->pooled; }
