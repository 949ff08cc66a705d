// mf_cnn.cu -- Mask R-CNN backbone (ResNet-101 + FPN) as wgmma tensor-core GEMMs (sm_90a).
//
// Replaces the dense-contraction part of the reference's Keras/TensorFlow sidecar
// (Core/Segmentation/MaskRCNN/MaskRCNN.py.in:55-58,101-111 -> matterport mrcnn `resnet_graph` +
// FPN top-down path; network source un-vendored, build.sh:278).  Every convolution is an
// implicit-GEMM  D[M x Cout] = A[M x K] * W[Cout x K]^T  with M = N*Hout*Wout output pixels,
// K = kh*kw*Cin, activations NHWC bf16, frozen BatchNorm + conv bias folded into the weights
// and a per-channel bias, residual add and ReLU fused into the epilogue.
//
// GEMM kernel (one 128 x BN output tile per CTA, three warpgroups = 384 threads):
//   warpgroup 0     TMA producer (one thread): cp.async.bulk.tensor.2d/3d (SWIZZLE_128B) A/B
//                   k-blocks of 64 into a 4-stage shared-memory ring, mbarrier expect_tx / complete_tx
//   warpgroups 1-2  consumers: each owns 64 rows of the tile and issues wgmma.mma_async m64nBNk16
//                   (bf16 in, fp32 accumulators in registers) straight from the swizzled ring slots;
//                   a slot is released (mbarrier arrive) once the wgmma group that read it has retired.
//                   Tile width BN = 128 when that still gives every SM a tile, else 64.
//                   Epilogue from registers: + bias, + residual, ReLU -> bf16 pairs to HBM
// 1x1 stride-1 convolutions feed the activation tensor straight to TMA (no im2col); 3x3 / stride 1
// convolutions use a 3-D tensor map (implicit GEMM); 7x7 and strided 1x1 go through a bf16 im2col buffer.
#include "mf_common.cuh"
#include "mf_kernels.h"
#include <cuda.h>
#include <cuda_bf16.h>
#include <vector>
#include <string>
#include <math.h>
#include <limits.h>
#include <stdlib.h>
#include <string.h>
#include <map>
#include <mutex>
#include <array>
#include <type_traits>

namespace mfb {

// ------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------
MF_D uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
MF_D void mbar_init(uint64_t* bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count)); }
MF_D void mbar_expect_tx(uint64_t* bar, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory"); }
MF_D void mbar_arrive(uint64_t* bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory"); }
MF_D void mbar_wait(uint64_t* bar, uint32_t parity)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "DONE:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
MF_D void tma_load_2d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1)
{
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
MF_D void tma_load_3d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1, int c2)
{
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
// shared-memory matrix descriptor (sm_90 wgmma): K-major operand, SWIZZLE_128B, rows of 128 B, 8-row groups 1024 B apart
MF_D uint64_t make_smem_desc(uint32_t saddr)
{
    uint64_t d = 0;
    d |= (uint64_t)((saddr & 0x3FFFF) >> 4);          // start address, 16-byte units          bits [0,14)
    d |= (uint64_t)1 << 16;                            // leading byte offset (unused for SW128 K-major) = 1
    d |= (uint64_t)(1024 >> 4) << 32;                  // stride byte offset: 8 rows x 128 B      bits [32,46)
    d |= (uint64_t)1 << 62;                            // layout type: SWIZZLE_128B               bits [62,64)
    return d;
}
MF_D void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
MF_D void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
MF_D void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// D[64 x N] += A[64 x 16] * B[N x 16]^T, both operands K-major in shared memory; scale-d = 1 (the accumulators start at zero)
#define WG_D8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define WG_D32(i) WG_D8(i), WG_D8(i + 8), WG_D8(i + 16), WG_D8(i + 24)
MF_D void wgmma_m64n64(float* d, uint64_t adesc, uint64_t bdesc)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\twgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
                 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
                 : WG_D32(0) : "l"(adesc), "l"(bdesc) : "memory");
}
MF_D void wgmma_m64n128(float* d, uint64_t adesc, uint64_t bdesc)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\twgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
                 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
                 : WG_D32(0), WG_D32(32) : "l"(adesc), "l"(bdesc) : "memory");
}
template <int BN>
MF_D void wgmma_tile(float (&d)[BN / 2], uint64_t adesc, uint64_t bdesc)
{
    if constexpr (BN == 128) wgmma_m64n128(d, adesc, bdesc);
    else wgmma_m64n64(d, adesc, bdesc);
}

// ------------------------------------------------------------------------------------------
// GEMM: out[M x N] (bf16) = relu?( A[M x K] * B[N x K]^T + bias[N] + residual[M x N] )
// ------------------------------------------------------------------------------------------
constexpr int GEMM_BM = 128, GEMM_BK = 64, GEMM_STAGES = 4, GEMM_THREADS = 384;   // 4 stages x 32 KB (BN = 128): one CTA per SM

// implicit-GEMM geometry of a 3x3 / stride 1 / pad 1 convolution: the A operand is the NHWC activation itself, seen through a 3-D
// tensor map (C, W, H); an M tile is a Wbox x Hbox pixel block (Wbox*Hbox = 128) and each of the 9 taps is the same block shifted
// by (kx-1, ky-1) -- TMA zero-fills the out-of-image part, which IS the padding.  No im2col buffer.
struct ConvGeom { int mode; int Wimg, Himg, Wbox, Hbox, cblocks; };

// OutT = __nv_bfloat16 (every backbone layer) or float (the RPN's 1x1 heads, whose scores feed a top-k: no bf16 ties)
template <int BN, typename OutT>
__global__ void __launch_bounds__(GEMM_THREADS, 1) k_gemm_bf16_wgmma(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
                                                                      const float* __restrict__ bias, const __nv_bfloat16* __restrict__ residual,
                                                                      OutT* __restrict__ out, int M, int N, int K, int relu, ConvGeom geo)
{
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // carve: [stages x A tile 16 KB][stages x B tile BN*128 B][barriers]
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    constexpr uint32_t A_BYTES = GEMM_BM * GEMM_BK * 2, B_BYTES = BN * GEMM_BK * 2;
    uint8_t* sA = smem;
    uint8_t* sB = smem + GEMM_STAGES * A_BYTES;
    uint64_t* full = (uint64_t*)(sB + GEMM_STAGES * B_BYTES);
    uint64_t* empty = full + GEMM_STAGES;

    const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
    const int tile_m = blockIdx.x, tile_n = blockIdx.y;
    const int num_k = K / GEMM_BK;
    int px0 = 0, py0 = 0;
    if (geo.mode) { const int tilesX = geo.Wimg / geo.Wbox; py0 = (tile_m / tilesX) * geo.Hbox; px0 = (tile_m % tilesX) * geo.Wbox; }

    if (threadIdx.x == 0) {
        for (int s = 0; s < GEMM_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], GEMM_THREADS - 128); }      // empty: one arrival per consumer thread
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (wg == 0) {
        if (t == 0) {
            // ===== TMA producer =====
            for (int kb = 0; kb < num_k; ++kb) {
                const int s = kb % GEMM_STAGES;
                const uint32_t ph = (kb / GEMM_STAGES) & 1;
                mbar_wait(&empty[s], ph ^ 1);
                mbar_expect_tx(&full[s], A_BYTES + B_BYTES);
                if (geo.mode) {
                    const int tap = kb / geo.cblocks, cb = kb - tap * geo.cblocks;
                    tma_load_3d(&mapA, &full[s], sA + s * A_BYTES, cb * GEMM_BK, px0 + tap % 3 - 1, py0 + tap / 3 - 1);
                } else
                    tma_load_2d(&mapA, &full[s], sA + s * A_BYTES, kb * GEMM_BK, tile_m * GEMM_BM);
                tma_load_2d(&mapB, &full[s], sB + s * B_BYTES, kb * GEMM_BK, tile_n * BN);
            }
        }
        return;
    }
    // ===== consumers: warpgroup c = wg - 1 owns tile rows [64 c, 64 c + 64) =====
    const int c = wg - 1;
    float d[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
    for (int kb = 0; kb < num_k; ++kb) {
        const int s = kb % GEMM_STAGES;
        mbar_wait(&full[s], (kb / GEMM_STAGES) & 1);
        const uint64_t adesc = make_smem_desc(smem_u32(sA + s * A_BYTES + c * 64 * 128));
        const uint64_t bdesc = make_smem_desc(smem_u32(sB + s * B_BYTES));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < GEMM_BK / 16; ++k)           // K = 16 bf16 = 32 bytes per wgmma: advance the start address by 2 (16-byte units)
            wgmma_tile<BN>(d, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k));
        wgmma_commit();
        wgmma_wait<1>();                                 // the group of k-block kb-1 has retired: its ring slot may be refilled
        if (kb > 0) mbar_arrive(&empty[(kb - 1) % GEMM_STAGES]);
    }
    wgmma_wait<0>();
    // ===== epilogue: accumulator fragment of m64nBN -- d[4j + 2h + e] is row 16 w + lane/4 + 8 h, column 8 j + 2 (lane%4) + e =====
    const int w = t >> 5, lane = t & 31;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int rt = c * 64 + w * 16 + (lane >> 2) + 8 * h;
        const int row = geo.mode ? (py0 + rt / geo.Wbox) * geo.Wimg + px0 + rt % geo.Wbox : tile_m * GEMM_BM + rt;
        if (row >= M) continue;
        OutT* optr = out + (size_t)row * N + tile_n * BN + 2 * (lane & 3);
        const __nv_bfloat16* rptr = residual ? residual + (size_t)row * N + tile_n * BN + 2 * (lane & 3) : nullptr;
        const float* bptr = bias + tile_n * BN + 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            const float2 b2 = __ldg(reinterpret_cast<const float2*>(bptr + 8 * j));
            float x0 = d[4 * j + 2 * h] + b2.x, x1 = d[4 * j + 2 * h + 1] + b2.y;
            if (rptr) { const __nv_bfloat162 r2 = *reinterpret_cast<const __nv_bfloat162*>(rptr + 8 * j); x0 += __low2float(r2); x1 += __high2float(r2); }
            if (relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
            if constexpr (std::is_same<OutT, float>::value) *reinterpret_cast<float2*>(optr + 8 * j) = make_float2(x0, x1);
            else *reinterpret_cast<__nv_bfloat162*>(optr + 8 * j) = __floats2bfloat162_rn(x0, x1);
        }
    }
}

// ------------------------------------------------------------------------------------------
// data-movement kernels around the GEMMs (NHWC bf16)
// ------------------------------------------------------------------------------------------
// im2col: A[m][(ky*kw + kx)*Cin + c], K padded with zeros to Kpad; 8 channels (16 B) per thread when Cin % 8 == 0
// nimg images stacked (the mask head's ROIs): row m = (img, oy, ox), each image padded on its own
__global__ void k_im2col(const __nv_bfloat16* __restrict__ in, int nimg, int Hin, int Win, int Cin, int Hout, int Wout, int kh, int kw, int stride,
                         int pad, int Kpad, __nv_bfloat16* __restrict__ A)
{
    const int K = kh * kw * Cin;
    const size_t total8 = (size_t)nimg * Hout * Wout * (Kpad / 8);
    for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total8; t += (size_t)gridDim.x * blockDim.x) {
        const int k8 = (int)(t % (Kpad / 8));
        const size_t m = t / (Kpad / 8);
        const int ox = (int)(m % Wout), oy = (int)((m / Wout) % Hout);
        const __nv_bfloat16* img = in + (m / ((size_t)Wout * Hout)) * Hin * Win * Cin;
        uint4 v = make_uint4(0, 0, 0, 0);
        const int k0 = k8 * 8;
        if ((Cin & 7) == 0) {
            if (k0 < K) {
                const int tap = k0 / Cin, c = k0 - tap * Cin;
                const int ky = tap / kw, kx = tap - ky * kw;
                const int iy = oy * stride - pad + ky, ix = ox * stride - pad + kx;
                if (iy >= 0 && iy < Hin && ix >= 0 && ix < Win) v = *reinterpret_cast<const uint4*>(img + ((size_t)iy * Win + ix) * Cin + c);
            }
        } else {
            __nv_bfloat16* e = reinterpret_cast<__nv_bfloat16*>(&v);
            for (int j = 0; j < 8; ++j) {
                const int k = k0 + j;
                if (k < K) {
                    const int tap = k / Cin, c = k - tap * Cin;
                    const int ky = tap / kw, kx = tap - ky * kw;
                    const int iy = oy * stride - pad + ky, ix = ox * stride - pad + kx;
                    if (iy >= 0 && iy < Hin && ix >= 0 && ix < Win) e[j] = img[((size_t)iy * Win + ix) * Cin + c];
                }
            }
        }
        *reinterpret_cast<uint4*>(A + m * Kpad + k0) = v;
    }
}
// 3x3 / stride 2 max pool, TensorFlow "same" padding (extra row/column at the END): window [2o, 2o+2] clipped
__global__ void k_maxpool3s2(const __nv_bfloat16* __restrict__ in, int Hin, int Win, int C, int Hout, int Wout, __nv_bfloat16* __restrict__ out)
{
    const size_t total = (size_t)Hout * Wout * C;
    for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
        const int c = (int)(t % C); const size_t p = t / C;
        const int ox = (int)(p % Wout), oy = (int)(p / Wout);
        float best = -INFINITY;
        for (int ky = 0; ky < 3; ++ky)
            for (int kx = 0; kx < 3; ++kx) {
                const int iy = 2 * oy + ky, ix = 2 * ox + kx;
                if (iy < Hin && ix < Win) best = fmaxf(best, __bfloat162float(in[((size_t)iy * Win + ix) * C + c]));
            }
        out[t] = __float2bfloat16(best);
    }
}
// FPN top-down: out = lateral + nearest-upsample2(top)
__global__ void k_upsample_add(const __nv_bfloat16* __restrict__ lateral, const __nv_bfloat16* __restrict__ top, int H, int W, int C,
                               __nv_bfloat16* __restrict__ out)
{
    const size_t total = (size_t)H * W * C;
    for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
        const int c = (int)(t % C); const size_t p = t / C;
        const int x = (int)(p % W), y = (int)(p / W);
        float v = __bfloat162float(lateral[t]) + __bfloat162float(top[((size_t)(y / 2) * (W / 2) + x / 2) * C + c]);
        out[t] = __float2bfloat16(v);
    }
}
// 1x1 / stride 2 sub-sampling (P6 = MaxPool 1x1 stride 2 of P5; also the A operand of strided 1x1 convolutions)
__global__ void k_subsample2(const __nv_bfloat16* __restrict__ in, int Hin, int Win, int C, __nv_bfloat16* __restrict__ out)
{
    const int Hout = Hin / 2, Wout = Win / 2;
    const size_t total8 = (size_t)Hout * Wout * (C / 8);
    for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total8; t += (size_t)gridDim.x * blockDim.x) {
        const int c8 = (int)(t % (C / 8)); const size_t p = t / (C / 8);
        const int ox = (int)(p % Wout), oy = (int)(p / Wout);
        *reinterpret_cast<uint4*>(out + p * C + c8 * 8) = *reinterpret_cast<const uint4*>(in + ((size_t)(2 * oy) * Win + 2 * ox) * C + c8 * 8);
    }
}
// R-MOLD (DESIGN §4) one axis: output sample o of the resized image reads input coordinate c = (o + 0.5) * zoom - 0.5, zoom = in / out,
// between taps i0 = floor(c) and i0 + 1 with weights w0 = 1 - (c - i0) and w1 = 1 - w0 (scipy.ndimage.zoom's arithmetic).  The file is
// built with FMA contraction on: the _rn intrinsics keep every step a separately rounded double operation.
MF_D void mold_axis(int o, double zoom, int& i0, double& w0, double& w1)
{
    const double c = __dsub_rn(__dmul_rn(__dadd_rn((double)o, 0.5), zoom), 0.5);
    const double f = floor(c);
    i0 = (int)f;
    w0 = __dsub_rn(1.0, __dsub_rn(c, f));
    w1 = __dsub_rn(1.0, w0);
}
// one channel of one resized sample: sum over the taps (y0,x0) (y0,x1) (y1,x0) (y1,x1) of (value * wy) * wx in that order, then truncated
// to uint8 (the resize's astype), then minus the mean pixel in float, rounded once to bf16
MF_D __nv_bfloat16 mold_value(int a, int b, int c, int d, double wy0, double wy1, double wx0, double wx1, float mean)
{
    double v = __dmul_rn(__dmul_rn((double)a, wy0), wx0);
    v = __dadd_rn(v, __dmul_rn(__dmul_rn((double)b, wy0), wx1));
    v = __dadd_rn(v, __dmul_rn(__dmul_rn((double)c, wy1), wx0));
    v = __dadd_rn(v, __dmul_rn(__dmul_rn((double)d, wy1), wx1));
    return __float2bfloat16((float)(int)v - mean);
}
// letter-boxed network input (R-MOLD): uint8 RGBA W x H -> bf16 NHWC S x S.  The image is resampled to newW x newH at (offx, offy) with
// taps outside the image reading 0; the padding is the uint8 value 0, so it becomes -MEAN_PIXEL.  One thread per output pixel, one grid row
// (blockIdx.y) per output row: no 64-bit index division
__global__ void k_mold_input(const uchar4* __restrict__ rgb, int W, int H, int S, double zoomx, double zoomy, int offx, int offy, int newW,
                             int newH, __nv_bfloat16* __restrict__ out)
{
    const float mr = 123.7f, mg = 116.8f, mb = 103.9f;      // MEAN_PIXEL (mrcnn config)
    const int y = blockIdx.y, x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= S) return;
    const int lx = x - offx, ly = y - offy;
    __nv_bfloat16* o = out + ((size_t)y * S + x) * 3;
    if (lx < 0 || lx >= newW || ly < 0 || ly >= newH) {
        o[0] = __float2bfloat16(-mr); o[1] = __float2bfloat16(-mg); o[2] = __float2bfloat16(-mb);
        return;
    }
    int x0, y0;
    double wx0, wx1, wy0, wy1;
    mold_axis(lx, zoomx, x0, wx0, wx1);
    mold_axis(ly, zoomy, y0, wy0, wy1);
    const uchar4 zero = make_uchar4(0, 0, 0, 0);
    const bool inx0 = x0 >= 0 && x0 < W, inx1 = x0 + 1 >= 0 && x0 + 1 < W, iny0 = y0 >= 0 && y0 < H, iny1 = y0 + 1 >= 0 && y0 + 1 < H;
    const uchar4 a = iny0 && inx0 ? rgb[(size_t)y0 * W + x0] : zero, b = iny0 && inx1 ? rgb[(size_t)y0 * W + x0 + 1] : zero;
    const uchar4 c = iny1 && inx0 ? rgb[(size_t)(y0 + 1) * W + x0] : zero, d = iny1 && inx1 ? rgb[(size_t)(y0 + 1) * W + x0 + 1] : zero;
    o[0] = mold_value(a.x, b.x, c.x, d.x, wy0, wy1, wx0, wx1, mr);
    o[1] = mold_value(a.y, b.y, c.y, d.y, wy0, wy1, wx0, wx1, mg);
    o[2] = mold_value(a.z, b.z, c.z, d.z, wy0, wy1, wx0, wx1, mb);
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// The GEMM launcher's process-wide state, behind one lock (handles may run on several threads and devices): the driver's
// cuTensorMapEncodeTiled, looked up once; and the tensor maps, which are pure functions of (pointer, geometry) -- the backbone's buffers
// never move, so every map is encoded once (first forward) and reused by all later launches.
static std::mutex g_gemmLock;
static PFN_encodeTiled g_encode = nullptr;
static std::map<std::array<uint64_t, 6>, CUtensorMap> g_mapCache;

static PFN_encodeTiled encode_fn()
{
    if (g_encode) return g_encode;
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn) throw CudaError{"cuTensorMapEncodeTiled not available"};
    return g_encode = (PFN_encodeTiled)fn;
}
// rank 2: row-major [rows x K] bf16, dims {K, rows}, box {64, boxRows}; rank 3: an NHWC activation, dims {C, W, H}, box {64, Wbox, Hbox}.
// SWIZZLE_128B.  Encoded on first use, then from the cache; under g_gemmLock
static CUtensorMap cached_map(const void* ptr, int rank, const cuuint64_t* dims, const cuuint32_t* box)
{
    const bool r3 = rank == 3;
    const std::array<uint64_t, 6> key = {(uint64_t)(uintptr_t)ptr, dims[0], dims[1], r3 ? dims[2] : 0, box[1], r3 ? box[2] : 0};
    auto it = g_mapCache.find(key);
    if (it != g_mapCache.end()) return it->second;
    const cuuint64_t strides[2] = {dims[0] * 2, dims[0] * dims[1] * 2};
    const cuuint32_t estr[3] = {1, 1, 1};
    CUtensorMap m;
    CUresult r = encode_fn()(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) throw CudaError{std::string(r3 ? "cuTensorMapEncodeTiled (3-D) failed: " : "cuTensorMapEncodeTiled failed: ") + std::to_string((int)r)};
    if (g_mapCache.size() < 4096) g_mapCache[key] = m;
    return m;
}

template <int BN>
static size_t gemm_smem_bytes() { return (size_t)GEMM_STAGES * (GEMM_BM * GEMM_BK * 2 + BN * GEMM_BK * 2) + 2 * GEMM_STAGES * 8 + 1024; }

void cnn_read_back(cudaStream_t s, void* dst, const void* src, size_t width, size_t rows, size_t pitch)
{
    if (!dst) return;
    cudaError_t e = cudaStreamSynchronize(s);
    if (e == cudaSuccess)
        e = rows == 1 ? cudaMemcpy(dst, src, width, cudaMemcpyDeviceToHost) : cudaMemcpy2D(dst, width, src, pitch, width, rows, cudaMemcpyDeviceToHost);
    cudaCheck(e, "download");
}

template <int BN, typename OutT>
static void launch_wgmma(const void* A, const void* B, const float* bias, const void* residual, void* out, int M, int N, int K, int relu,
                         cudaStream_t s, const ConvGeom& geo, int Cin)
{
    // the dynamic shared memory this instantiation is opted in for: the attribute belongs to a (function, device) pair
    static PerDevice<size_t> smem([](int) {
        cudaCheck(cudaFuncSetAttribute(k_gemm_bf16_wgmma<BN, OutT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gemm_smem_bytes<BN>()),
                  "cudaFuncSetAttribute");
        return gemm_smem_bytes<BN>();
    });
    const size_t smemBytes = smem.get();
    const cuuint64_t dimsA[3] = {(cuuint64_t)(geo.mode ? Cin : K), (cuuint64_t)(geo.mode ? geo.Wimg : M), (cuuint64_t)geo.Himg}, dimsB[2] = {(cuuint64_t)K, (cuuint64_t)N};
    const cuuint32_t boxA[3] = {64, (cuuint32_t)(geo.mode ? geo.Wbox : GEMM_BM), (cuuint32_t)geo.Hbox}, boxB[2] = {64, BN};
    CUtensorMap mA, mB;
    {
        std::lock_guard<std::mutex> lock(g_gemmLock);
        mA = cached_map(A, geo.mode ? 3 : 2, dimsA, boxA);
        mB = cached_map(B, 2, dimsB, boxB);
    }
    launch(Enq{s, nullptr}, nullptr, k_gemm_bf16_wgmma<BN, OutT>, dim3((M + GEMM_BM - 1) / GEMM_BM, N / BN), dim3(GEMM_THREADS), smemBytes,
           mA, mB, bias, (const __nv_bfloat16*)residual, (OutT*)out, M, N, K, relu, geo);
}

// D = relu?(A * B^T + bias + residual); all device pointers; K % 64 == 0, N % 64 == 0
// conv3x3 != nullptr: A is an NHWC activation [Himg x Wimg x Cin] and the GEMM is the implicit 3x3/s1/p1 convolution (K = 9*Cin)
// outF32: D is written as fp32 (residual must then be null), else as bf16
void launch_gemm_bf16(const void* A, const void* B, const float* bias, const void* residual, void* out, int M, int N, int K, int relu, cudaStream_t s,
                      const int* conv3x3 /* Wimg, Himg, Cin */, bool outF32)
{
    // every refusal comes before the first driver call
    if (outF32 && residual) throw CudaError{"gemm: the fp32 output takes no residual"};
    ConvGeom geo; memset(&geo, 0, sizeof geo);
    if (conv3x3) {
        const int Wimg = conv3x3[0], Himg = conv3x3[1], Cin = conv3x3[2];
        if (!cnn_conv_implicit(3, 1, 1, Cin, Himg, Wimg) || K != 9 * Cin || M != Wimg * Himg) throw CudaError{"conv3x3: unsupported geometry"};
        geo.mode = 1; geo.Wimg = Wimg; geo.Himg = Himg; geo.Wbox = Wimg >= 128 ? 128 : Wimg; geo.Hbox = 128 / geo.Wbox; geo.cblocks = Cin / 64;
    }
    if (K <= 0 || N <= 0 || M <= 0 || K % 64 || N % 64) throw CudaError{"gemm: need M > 0, and K > 0 and N > 0 multiples of 64"};
    const int mtiles = (M + GEMM_BM - 1) / GEMM_BM, Cin = conv3x3 ? conv3x3[2] : 0;
    // fill the machine: with few M tiles prefer the narrow N tile (twice the CTAs)
    const bool wide = N % 128 == 0 && mtiles * (N / 128) >= num_sms();
    if (outF32) {
        if (wide) launch_wgmma<128, float>(A, B, bias, residual, out, M, N, K, relu, s, geo, Cin);
        else launch_wgmma<64, float>(A, B, bias, residual, out, M, N, K, relu, s, geo, Cin);
    } else {
        if (wide) launch_wgmma<128, __nv_bfloat16>(A, B, bias, residual, out, M, N, K, relu, s, geo, Cin);
        else launch_wgmma<64, __nv_bfloat16>(A, B, bias, residual, out, M, N, K, relu, s, geo, Cin);
    }
}

// ---- backbone ---------------------------------------------------------------------------
struct Backbone {
    int S;                                    // square network input (1024)
    cudaStream_t stream;
    std::vector<LayerGeom> layers;            // the table's: conv1, per block branch2a, 2b, 2c (+ branch1 in block a), 4 laterals, 4 outputs
    WeightStore w;
    DevBuf<__nv_bfloat16> input, bufA, bufB, bufC, bufS, col, C2, C3, C4, C5, P[5], lat, td;
    double flops = 0;
    int gemms = 0;
    Backbone(int S, unsigned seed, cudaStream_t s);
};

// geometry rule of the implicit 3x3 path, the only one (launch_gemm_bf16 refuses exactly what it refuses): the Wbox x Hbox TMA box of
// 128 pixels (Wbox = min(W, 128), Hbox = 128 / Wbox) must tile the image exactly, since the producer expects a full 16 KiB A tile per
// k-block and a smaller box would never complete the barrier.  Admitted: W a divisor of 128 of at least 8 with H % (128 / W) == 0, or
// W a multiple of 128 (up to 128 Ki); Cin a positive multiple of 64; M = H * W within int
bool cnn_conv_implicit(int k, int stride, int pad, int Cin, int Hin, int Win)
{
    if (k != 3 || stride != 1 || pad != 1 || Cin <= 0 || Cin % 64 || Cin > INT_MAX / 9 || Hin <= 0 || Win <= 0 || Win > 128 * 1024 ||
        Hin > INT_MAX / Win)
        return false;
    const int wbox = Win >= 128 ? 128 : Win;
    return wbox >= 8 && 128 % wbox == 0 && Win % wbox == 0 && Hin % (128 / wbox) == 0;
}

// runs convolution L (weights W [rows x K], bias B) on in[Hin x Win x cin] -> out[Hout x Wout x rows]; col: im2col scratch
static void conv_layer(const LayerGeom& L, const __nv_bfloat16* W, const float* B, __nv_bfloat16* col, const __nv_bfloat16* in, int Hin, int Win,
                       __nv_bfloat16* out, const __nv_bfloat16* residual, int relu, cudaStream_t s, int* HoutP, int* WoutP)
{
    const int Hout = (Hin + 2 * L.pad - L.k) / L.stride + 1, Wout = (Win + 2 * L.pad - L.k) / L.stride + 1;
    const int M = Hout * Wout;
    const __nv_bfloat16* A = in;
    if (HoutP) *HoutP = Hout;
    if (WoutP) *WoutP = Wout;
    if (cnn_conv_implicit(L.k, L.stride, L.pad, L.cin, Hin, Win)) {
        int g3[3] = {Win, Hin, L.cin};
        launch_gemm_bf16(in, W, B, residual, out, M, L.rows, L.K, relu, s, g3);
        return;
    }
    if (!(L.k == 1 && L.stride == 1)) {
        if (L.k == 1 && L.stride == 2 && (L.cin % 8) == 0)
            launch(Enq{s, nullptr}, nullptr, k_subsample2, 4 * num_sms(), 256, 0, in, Hin, Win, L.cin, col);
        else
            launch_im2col(in, 1, Hin, Win, L.cin, Hout, Wout, L.k, L.stride, L.pad, L.K, col, s);
        A = col;
    }
    launch_gemm_bf16(A, W, B, residual, out, M, L.rows, L.K, relu, s);
}

// runs backbone layer li on in[Hin x Win x Cin] -> out[Hout x Wout x Cout]
static void run_conv(Backbone* b, int li, const __nv_bfloat16* in, int Hin, int Win, __nv_bfloat16* out, const __nv_bfloat16* residual, int relu,
                     cudaStream_t s, int* HoutP = nullptr, int* WoutP = nullptr)
{
    const LayerGeom& L = b->layers[li];
    int Hout, Wout;
    conv_layer(L, b->w.w(li), b->w.b(li), b->col, in, Hin, Win, out, residual, relu, s, &Hout, &Wout);
    b->flops += 2.0 * Hout * Wout * (double)L.rows * (double)(L.k * L.k * L.cin);
    b->gemms++;
    if (HoutP) *HoutP = Hout;
    if (WoutP) *WoutP = Wout;
}

void launch_im2col(const void* in, int nimg, int Hin, int Win, int Cin, int Hout, int Wout, int k, int stride, int pad, int Kpad, void* col, cudaStream_t s)
{
    launch(Enq{s, nullptr}, nullptr, k_im2col, 8 * num_sms(), 256, 0, (const __nv_bfloat16*)in, nimg, Hin, Win, Cin, Hout, Wout, k, k, stride, pad, Kpad,
           (__nv_bfloat16*)col);
}

// mould_image's letter box as mf_backbone_mold applies it (the detection heads map boxes back through the same geometry)
MoldGeom cnn_mold_geometry(int S, int W, int H)
{
    MoldGeom g;
    g.scale = fminf((float)S / (float)W, (float)S / (float)H);
    g.newW = (int)lroundf(W * g.scale); g.newH = (int)lroundf(H * g.scale);
    g.offx = (S - g.newW) / 2; g.offy = (S - g.newH) / 2;
    return g;
}

// a convolution whose weights are not in the backbone's table (the RPN's shared 3x3): the same path as the backbone's layers
void cnn_conv(const void* in, int Hin, int Win, int Cin, int Cout, int k, int stride, int pad, const void* W, const float* B, void* col, void* out, int relu,
              cudaStream_t s)
{
    const LayerGeom L = {Cin, Cout, k, stride, pad, (k * k * Cin + 63) / 64 * 64};
    conv_layer(L, (const __nv_bfloat16*)W, B, (__nv_bfloat16*)col, (const __nv_bfloat16*)in, Hin, Win, (__nv_bfloat16*)out, nullptr, relu, s, nullptr,
               nullptr);
}

}  // namespace mfb

using namespace mfb;

// ==========================================================================================
// the backbone handle
// ==========================================================================================
struct mf_backbone : Backbone { using Backbone::Backbone; };

// ResNet-101-FPN (mf_weights.cu has the layer table); throws CudaError
Backbone::Backbone(int S_, unsigned seed, cudaStream_t s) : S(S_), stream(s), w(MRCNN_BACKBONE, seed, s)
{
    for (int i = 0; i < mrcnn_num_layers(MRCNN_BACKBONE); ++i) layers.push_back(mrcnn_layer(MRCNN_BACKBONE, i));
    const size_t big = (size_t)(S / 2) * (S / 2) * 64;                         // stem output == largest activation (elements): C1 512x512x64 = C2 256x256x256
    input.alloc((size_t)S * S * 3);
    bufA.alloc(big); bufB.alloc(big); bufC.alloc(big); bufS.alloc(big);
    col.alloc((size_t)(S / 4) * (S / 4) * 9 * 256);                            // largest im2col: FPN P2 3x3 on 256x256x256 (and C2 3x3 64ch is smaller); stem: 512*512*192
    const int fs[4] = {S / 4, S / 8, S / 16, S / 32};
    C2.alloc((size_t)fs[0] * fs[0] * 256); C3.alloc((size_t)fs[1] * fs[1] * 512); C4.alloc((size_t)fs[2] * fs[2] * 1024); C5.alloc((size_t)fs[3] * fs[3] * 2048);
    for (int i = 0; i < 4; ++i) P[i].alloc((size_t)fs[i] * fs[i] * 256);
    P[4].alloc((size_t)(fs[3] / 2) * (fs[3] / 2) * 256);
    lat.alloc((size_t)fs[0] * fs[0] * 256); td.alloc((size_t)fs[0] * fs[0] * 256);
}

namespace mfb {
cudaStream_t backbone_stream(mf_backbone* h) { return h->stream; }
const void* backbone_input(mf_backbone* h) { return h->input; }

void* backbone_level(mf_backbone* h, int level, int* dims3)
{
    const int S = h->S;
    const int fs[5] = {S / 4, S / 8, S / 16, S / 32, S / 64};
    const int cdim[4] = {256, 512, 1024, 2048};
    if (level >= 0 && level < 4) { dims3[0] = dims3[1] = fs[level]; dims3[2] = cdim[level]; __nv_bfloat16* c[4] = {h->C2, h->C3, h->C4, h->C5}; return c[level]; }
    if (level >= 4 && level < 9) { dims3[0] = dims3[1] = fs[level - 4]; dims3[2] = 256; return h->P[level - 4]; }
    return nullptr;
}

// letter-box + normalise a 640x480 (or any) RGBA8 device image into the network input (MaskRCNN.py.in mold_inputs; rule R-MOLD)
void backbone_mold(mf_backbone* h, const void* d_rgba, int W, int H)
{
    const int S = h->S;
    const MoldGeom g = cnn_mold_geometry(S, W, H);
    const double zoomx = (double)W / (double)g.newW, zoomy = (double)H / (double)g.newH;     // in / out per axis (R-MOLD)
    if (S > 65535) throw CudaError{"mold: the input size exceeds the grid's 65535 rows"};
    launch(Enq{h->stream, nullptr}, nullptr, k_mold_input, dim3((S + 255) / 256, S), 256, 0, (const uchar4*)d_rgba, W, H, S, zoomx, zoomy, g.offx,
           g.offy, g.newW, g.newH, h->input.p);
}

// forward on an already-moulded input (device, NHWC bf16 S x S x 3).  Outputs stay on the device (P2..P6, NHWC bf16).
void backbone_forward(mf_backbone* h, const void* d_input)
{
    Backbone* b = h; cudaStream_t s = h->stream;
    const Enq q{s, nullptr};
    b->flops = 0; b->gemms = 0;
    const int S = b->S;
    int H, W;
    int li = 0;                                      // the next layer of the table
    // C1: 7x7/2 + ReLU, max-pool 3x3/2
    run_conv(b, li++, (const __nv_bfloat16*)d_input, S, S, b->bufA, nullptr, 1, s, &H, &W);
    launch(q, nullptr, k_maxpool3s2, 8 * num_sms(), 256, 0, b->bufA.p, H, W, 64, H / 2, W / 2, b->bufB.p);
    H /= 2; W /= 2;
    __nv_bfloat16* x = b->bufB;                      // current block input
    const int nblocks[4] = {3, 4, 23, 3};
    __nv_bfloat16* stageOut[4] = {b->C2, b->C3, b->C4, b->C5};
    for (int st = 0; st < 4; ++st)
        for (int blk = 0; blk < nblocks[st]; ++blk) {
            const int c1 = li, c2 = li + 1, c3 = li + 2, sc = blk == 0 ? li + 3 : -1;
            li += blk == 0 ? 4 : 3;
            // pick three scratch buffers different from x
            __nv_bfloat16* t[3]; int n = 0;
            __nv_bfloat16* all[4] = {b->bufA, b->bufB, b->bufC, b->bufS};
            for (int k = 0; k < 4 && n < 3; ++k) if (all[k] != x) t[n++] = all[k];
            int H1, W1;
            run_conv(b, c1, x, H, W, t[0], nullptr, 1, s, &H1, &W1);
            run_conv(b, c2, t[0], H1, W1, t[1], nullptr, 1, s);
            const __nv_bfloat16* shortcut = x;
            if (sc >= 0) { run_conv(b, sc, x, H, W, t[2], nullptr, 0, s); shortcut = t[2]; }
            const bool last = blk == nblocks[st] - 1;
            __nv_bfloat16* y = last ? stageOut[st] : t[0];
            run_conv(b, c3, t[1], H1, W1, y, shortcut, 1, s);
            x = y; H = H1; W = W1;
        }
    // FPN
    const int fs[4] = {S / 4, S / 8, S / 16, S / 32};
    __nv_bfloat16* Cs[4] = {b->C2, b->C3, b->C4, b->C5};
    const int fpnLat = li, fpnOut = li + 4;
    // P5 lateral
    run_conv(b, fpnLat + 3, Cs[3], fs[3], fs[3], b->td, nullptr, 0, s);
    __nv_bfloat16* top = b->td;                       // running top-down map (pre-3x3)
    __nv_bfloat16* tdBuf[2] = {b->bufA, b->bufB};
    run_conv(b, fpnOut + 3, top, fs[3], fs[3], b->P[3], nullptr, 0, s);
    for (int i = 2; i >= 0; --i) {
        run_conv(b, fpnLat + i, Cs[i], fs[i], fs[i], b->lat, nullptr, 0, s);
        __nv_bfloat16* nt = tdBuf[i & 1];
        launch(q, nullptr, k_upsample_add, 8 * num_sms(), 256, 0, b->lat.p, top, fs[i], fs[i], 256, nt);
        top = nt;
        run_conv(b, fpnOut + i, top, fs[i], fs[i], b->P[i], nullptr, 0, s);
    }
    launch(q, nullptr, k_subsample2, 64, 256, 0, b->P[3].p, fs[3], fs[3], 256, b->P[4].p);       // P6
}
}  // namespace mfb

// ==========================================================================================
// C ABI (declared in include/maskfusion_b200.h)
// ==========================================================================================
extern "C" int mf_gemm_bf16(const void* dA, const void* dB, const float* dBias, const void* dResidual, void* dOut, int M, int N, int K, int relu, void* stream)
{
    MF_TRY
    launch_gemm_bf16(dA, dB, dBias, dResidual, dOut, M, N, K, relu, (cudaStream_t)stream);
    return 0;
    MF_CATCH(-2)
}

// implicit-GEMM 3x3 / stride 1 / pad 1 convolution on an NHWC bf16 activation (weights [Cout][3][3][Cin] bf16); the geometry is
// cnn_conv_implicit's, anything else returns -2 before a driver call
extern "C" int mf_conv3x3_bf16(const void* dIn, const void* dW, const float* dBias, const void* dResidual, void* dOut, int H, int W, int Cin, int Cout,
                               int relu, void* stream)
{
    MF_TRY
    int g3[3] = {W, H, Cin};
    // products in unsigned arithmetic: a refused geometry may overflow them, and the refusal does not read them
    launch_gemm_bf16(dIn, dW, dBias, dResidual, dOut, (int)((unsigned)H * (unsigned)W), Cout, (int)(9u * (unsigned)Cin), relu, (cudaStream_t)stream, g3);
    return 0;
    MF_CATCH(-2)
}

extern "C" mf_backbone* mf_backbone_create(int input_size, unsigned seed, void* stream)
{
    MF_TRY
    if (input_size % 64) { mf_set_error("input size must be a multiple of 64 (mrcnn: IMAGE_MAX_DIM=1024)"); return nullptr; }
    return new mf_backbone(input_size, seed, (cudaStream_t)stream);
    MF_CATCH_AS(nullptr, "backbone: ")
}

extern "C" void mf_backbone_destroy(mf_backbone* h) { delete h; }

extern "C" int mf_backbone_num_layers(mf_backbone* h)
{
    MF_TRY
    if (!h) throw CudaError{"backbone: null handle"};
    return (int)h->layers.size();
    MF_CATCH(-1)
}
// layer table: Cin Cout k stride pad Kpad
extern "C" int mf_backbone_layer(mf_backbone* h, int i, int* out6)
{
    MF_TRY
    if (!h || i < 0 || i >= (int)h->layers.size() || !out6) throw CudaError{"backbone: bad layer index"};
    const LayerGeom& L = h->layers[i];
    out6[0] = L.cin; out6[1] = L.rows; out6[2] = L.k; out6[3] = L.stride; out6[4] = L.pad; out6[5] = L.K;
    return 0;
    MF_CATCH(-1)
}
// weights [Cout x Kpad] fp32 (bf16-representable), (ky,kx,cin) order along K; bias [Cout]
extern "C" int mf_backbone_get_weights(mf_backbone* h, int i, float* w, float* bias)
{
    MF_TRY
    if (!h) throw CudaError{"backbone: null handle"};
    h->w.get(i, w, bias);
    return 0;
    MF_CATCH(-1)
}

// pretrained weights (mf_weights.cu): every layer is read, checked and folded on the host before the device tables change; the copy is
// ordered on the handle's stream and complete on return
extern "C" int mf_backbone_load_weights(mf_backbone* h, const char* path)
{
    MF_TRY
    if (!h) throw CudaError{"backbone: null handle"};
    h->w.load(path, h->stream);
    return 0;
    MF_CATCH(-1)
}

extern "C" int mf_backbone_forward(mf_backbone* h, const void* d_input)
{
    MF_TRY
    if (!h) throw CudaError{"backbone: null handle"};
    backbone_forward(h, d_input);
    return 0;
    MF_CATCH(-1)
}
extern "C" double mf_backbone_flops(mf_backbone* h) { return h ? h->flops : 0; }
extern "C" int mf_backbone_num_gemms(mf_backbone* h) { return h ? h->gemms : 0; }
extern "C" void* mf_backbone_input_buffer(mf_backbone* h) { return h ? h->input.p : nullptr; }
extern "C" void* mf_backbone_stream(mf_backbone* h) { return h ? (void*)h->stream : nullptr; }
// level 0..3 = C2..C5, 4..8 = P2..P6; returns device pointer, fills dims (H, W, C)
extern "C" void* mf_backbone_output(mf_backbone* h, int level, int* dims3) { return h ? backbone_level(h, level, dims3) : nullptr; }
extern "C" int mf_backbone_download(mf_backbone* h, int level, void* host_bf16)
{
    MF_TRY
    int d[3];
    const void* p = h ? backbone_level(h, level, d) : nullptr;
    if (!p) throw CudaError{"backbone: no handle or level outside 0..8"};
    cnn_read_back(h->stream, host_bf16, p, (size_t)d[0] * d[1] * d[2] * 2);
    return 0;
    MF_CATCH(-1)
}
extern "C" int mf_backbone_mold(mf_backbone* h, const void* d_rgba, int W, int H)
{
    MF_TRY
    if (!h) throw CudaError{"backbone: null handle"};
    if (W <= 0 || H <= 0) throw CudaError{"mold: the image needs W > 0 and H > 0"};
    backbone_mold(h, d_rgba, W, H);
    return 0;
    MF_CATCH(-1)
}
