// mf_track.cu -- dense RGB-D odometry on the device (sm_90a).
//   ICP point-to-plane JtJ/Jtr   <- icpKernel / ICPReduction,        Core/Cuda/reduce.cu:259-444
//   photometric correspondences  <- residualKernel / RGBResidual,   reduce.cu:774-997
//   photometric JtJ/Jtr          <- rgbKernel / RGBReduction,        reduce.cu:529-713
//   SO(3) pre-alignment          <- so3Kernel / SO3Reduction,        reduce.cu:999-1202
//   Gauss-Newton driver          <- RGBDOdometry::getIncrementalTransformation, RGBDOdometry.cpp:227-497
//                                   + OdometryProvider::{rodrigues,computeUpdateSE3}, OdometryProvider.h:32-90
//
// The reference returns to the host after every one of its <= 67 kernel pairs per model per
// frame (cudaDeviceSynchronize + 116-byte D2H + Eigen LDLT).  Here the whole schedule of a
// frame -- SO(3) pre-alignment, then pyramid levels 2, 1, 0 -- is ONE cooperative launch,
// k_track_persistent: one CTA per SM, the CTAs split between the tracked models (a flat grid,
// CTA ranges per model), so N objects on one GPU share the launch.  Every reduction exchanges
// one fp64 partial row per CTA as flagged words; each CTA then sums all rows of its model in
// fixed order and runs the same 6x6 solve (pivoted LDLT, double), so the solver state is
// replicated bit for bit without a broadcast.  Results are deterministic for a fixed launch shape.
// MFB200_TRACK_CACHE=1 keeps the pose-independent pixel inputs of a level in shared memory (same bits).
// k_icp_only is a stand-alone ICP reduction at a given pose (last-block ticket) for the parity tests.
#include "mf_common.cuh"
#include "mf_kernels.h"
#include "mf_host.h"
#include <float.h>
#include <algorithm>
#include <stdlib.h>
#include <string>

namespace mfb {

// per-level shared-memory cache of the pose-independent pixel inputs (A/B environment switch MFB200_TRACK_CACHE; see launch_tracking)
#ifndef MFB200_DEFAULT_TRACK_CACHE
#define MFB200_DEFAULT_TRACK_CACHE 0
#endif
#define CACHE_BYTES_PER_SLOT 44        // float4 vertex + float4 normal + depth + packed (valid, intensity, x, y) + Sobel gradient
#define TRK_THREADS 256
#define NACC_ICP 29
#define NACC_RGB 27
#define NACC (NACC_ICP + NACC_RGB)

MF_D float3 m3v(const float* R, float3 v)
{
    return make_float3((R[0] * v.x + R[1] * v.y) + R[2] * v.z, (R[3] * v.x + R[4] * v.y) + R[5] * v.z, (R[6] * v.x + R[7] * v.y) + R[8] * v.z);
}

// ---------------------------------------------------------------------------------------
// small dense maths (single thread, double)
// ---------------------------------------------------------------------------------------
__device__ void ldltSolve(const double* Ain, const double* b, int n, double* x)
{
    // pivoted LDL^T with Eigen's conventions: pivot on the largest remaining diagonal,
    // pivots <= DBL_MIN contribute 0 to the solution (RGBDOdometry.cpp:313,451-459)
    double A[36], y[6]; int perm[6];
    for (int i = 0; i < n * n; ++i) A[i] = Ain[i];
    for (int i = 0; i < n; ++i) perm[i] = i;
    int kend = n;
    for (int k = 0; k < n; ++k) {
        int piv = k; double best = fabs(A[k * n + k]);
        for (int i = k + 1; i < n; ++i) if (fabs(A[i * n + i]) > best) { best = fabs(A[i * n + i]); piv = i; }
        if (piv != k) {
            for (int j = 0; j < n; ++j) { double t = A[k * n + j]; A[k * n + j] = A[piv * n + j]; A[piv * n + j] = t; }
            for (int j = 0; j < n; ++j) { double t = A[j * n + k]; A[j * n + k] = A[j * n + piv]; A[j * n + piv] = t; }
            int t = perm[k]; perm[k] = perm[piv]; perm[piv] = t;
        }
        double d = A[k * n + k];
        if (fabs(d) <= DBL_MIN) { kend = k; break; }
        for (int i = k + 1; i < n; ++i) A[i * n + k] /= d;
        for (int i = k + 1; i < n; ++i)
            for (int j = k + 1; j <= i; ++j) {
                A[i * n + j] -= A[i * n + k] * d * A[j * n + k];
                A[j * n + i] = A[i * n + j];
            }
    }
    for (int i = 0; i < n; ++i) y[i] = b[perm[i]];
    for (int i = 0; i < n; ++i) for (int j = 0; j < i && j < kend; ++j) y[i] -= A[i * n + j] * y[j];
    for (int i = 0; i < n; ++i) {
        double d = (i < kend) ? A[i * n + i] : 0.0;
        y[i] = (fabs(d) > DBL_MIN) ? y[i] / d : 0.0;
    }
    for (int i = n - 1; i >= 0; --i) for (int j = i + 1; j < n; ++j) if (i < kend) y[i] -= A[j * n + i] * y[j];
    for (int i = 0; i < n; ++i) x[perm[i]] = y[i];
}

// R-SINCOS (DESIGN.md): one fixed Taylor polynomial (Horner, no contraction: this file is compiled -fmad=false) for the tiny update
// angles of the Gauss-Newton steps, the same on both sides of the parity contract (oracle/orc_odometry.c: orc_det_sincos);
// the library beyond |x| = 0.8 (never reached by a converging tracker).
__device__ __forceinline__ void detSincos(double x, double* s, double* c)
{
    if (!(fabs(x) <= 0.8)) { sincos(x, s, c); return; }
    const double z = x * x;
    double ps = -1.0 / 51090942171709440000.0;
    ps = ps * z + 1.0 / 121645100408832000.0;
    ps = ps * z - 1.0 / 355687428096000.0;
    ps = ps * z + 1.0 / 1307674368000.0;
    ps = ps * z - 1.0 / 6227020800.0;
    ps = ps * z + 1.0 / 39916800.0;
    ps = ps * z - 1.0 / 362880.0;
    ps = ps * z + 1.0 / 5040.0;
    ps = ps * z - 1.0 / 120.0;
    ps = ps * z + 1.0 / 6.0;
    *s = x - x * (z * ps);
    double pc = 1.0 / 2432902008176640000.0;
    pc = pc * z - 1.0 / 6402373705728000.0;
    pc = pc * z + 1.0 / 20922789888000.0;
    pc = pc * z - 1.0 / 87178291200.0;
    pc = pc * z + 1.0 / 479001600.0;
    pc = pc * z - 1.0 / 3628800.0;
    pc = pc * z + 1.0 / 40320.0;
    pc = pc * z - 1.0 / 720.0;
    pc = pc * z + 1.0 / 24.0;
    pc = pc * z - 1.0 / 2.0;
    *c = 1.0 + z * pc;
}

MF_D double shflD(double v, int src)
{
    int lo = __double2loint(v), hi = __double2hiint(v);
    lo = __shfl_sync(0xffffffffu, lo, src); hi = __shfl_sync(0xffffffffu, hi, src);
    return __hiloint2double(hi, lo);
}

// N x N (N = 3 or 6) symmetric system by ONE WARP with exactly the arithmetic of the sequential pivoted LDL^T above (= the oracle's
// orc_ldlt_solve = Eigen's conventions): lane i < N keeps row i of the FULL matrix in registers; pivot search, symmetric row/column
// swap, column scaling (IEEE division), trailing update A[i][j] -= (A[i][k] * d) * A[j][k], symmetric fill, the two substitutions --
// every element sees the same operations in the same order as in the sequential routine, so the solution is BIT-IDENTICAL to it
// (parity contract: with fp64 sums that round to the oracle's floats, the whole Gauss-Newton trajectory is reproduced bit for bit).
// All 32 lanes must call; A (N*N, row-major) and b (N) are read from shared memory, x (N) is written there.
// Register-fed core: lane i < N passes row i of the matrix in a[] and b[i] in bOwn (idle lanes mirror row N - 1).
template <int N>
MF_D void ldltSolvePivWarpRegs(double (&a)[N], double bOwn, double* x)
{
    const int lane = threadIdx.x & 31;
    const bool act = lane < N;
    const int r = act ? lane : N - 1;                      // idle lanes mirror the last row; they only ever supply nothing
    int perm = r;
    int kend = N;
#pragma unroll
    for (int k = 0; k < N; ++k) {
        if (k < kend) {                                    // warp uniform
            double dg = a[0];                              // this lane's diagonal entry A[r][r]
#pragma unroll
            for (int j = 1; j < N; ++j) if (r == j) dg = a[j];
            int piv = k; double best = fabs(shflD(dg, k));
#pragma unroll
            for (int i = k + 1; i < N; ++i) { const double v = fabs(shflD(dg, i)); if (v > best) { best = v; piv = i; } }
            if (piv != k) {                                // warp uniform
                const int src = lane == k ? piv : (lane == piv ? k : lane);
#pragma unroll
                for (int j = 0; j < N; ++j) a[j] = shflD(a[j], src);                  // rows k <-> piv
                perm = __shfl_sync(0xffffffffu, perm, src);
                const double ak = a[k];
                double ap = ak;
#pragma unroll
                for (int q = k + 1; q < N; ++q) if (piv == q) ap = a[q];
                a[k] = ap;                                                          // columns k <-> piv
#pragma unroll
                for (int q = k + 1; q < N; ++q) if (piv == q) a[q] = ak;
            }
            const double d = shflD(a[k], k);
            if (fabs(d) <= DBL_MIN) kend = k;
            else {
                if (act && lane > k) a[k] = a[k] / d;
                // Trailing update of BOTH halves, each entry with the sequential routine's operand order: the lower entry (i, j <= i) is
                // A[i][j] - (A[i][k] * d) * A[j][k]; the upper entry (i, j > i) mirrors the lower entry (j, i) = A[j][i] - (A[j][k] * d) * A[i][k],
                // so it is evaluated as exactly that product.  The two halves therefore stay bit-identical without the copy
                // A[j][i] = A[i][j] of the sequential routine (which cost 2 shuffles per pair here).
                const double ad = a[k] * d;
#pragma unroll
                for (int j = k + 1; j < N; ++j) {
                    const double cj = shflD(a[k], j);                               // A[j][k] (scaled)
                    const double lo = a[j] - ad * cj, up = a[j] - (cj * d) * a[k];
                    if (act && lane > k) a[j] = (j <= lane) ? lo : up;
                }
            }
        }
    }
    if (kend < N) {
#pragma unroll
        for (int j = 0; j < N; ++j) if (act && lane >= kend && j >= kend && j < lane) a[j] = 0.0;
    }
    double dg = a[0];                                      // this lane's pivot d_r
#pragma unroll
    for (int j = 1; j < N; ++j) if (r == j) dg = a[j];
    double y = shflD(bOwn, perm);                          // b[perm]: the right-hand side of the row this lane now holds
#pragma unroll
    for (int j = 0; j < N - 1; ++j) {
        const double yj = shflD(y, j);
        if (act && lane > j && j < kend) y = y - a[j] * yj;
    }
    {
        const double dd = lane < kend ? dg : 0.0;
        y = (fabs(dd) > DBL_MIN) ? y / dd : 0.0;
    }
    // L^T x = z.  Row i of L^T is column i of L: L[j][i] = (entry (j, i) before its scaling) / d_i, and that unscaled value is what
    // this lane's own UPPER entry (i, j) still holds (it was last touched at step i - 1).  Same operands, same division => same bits
    // as the stored factor, and no shuffles of the factor.
    double lt[N];
#pragma unroll
    for (int j = 1; j < N; ++j) lt[j] = a[j] / dg;
    double yf[N];
    yf[N - 1] = shflD(y, N - 1);
#pragma unroll
    for (int i = N - 2; i >= 0; --i) {
        if (lane == i && i < kend) {
#pragma unroll
            for (int j = i + 1; j < N; ++j) y = y - lt[j] * yf[j];                  // ascending j, as the sequential loop
        }
        yf[i] = shflD(y, i);
    }
    if (act) x[perm] = y;
    __syncwarp();
}
template <int N>
MF_D void ldltSolvePivWarp(const double* __restrict__ A, const double* __restrict__ b, double* x)
{
    const int lane = threadIdx.x & 31;
    const int r = lane < N ? lane : N - 1;
    double a[N];
#pragma unroll
    for (int j = 0; j < N; ++j) a[j] = A[r * N + j];
    ldltSolvePivWarpRegs<N>(a, b[r], x);
}

__device__ void rodrigues(const double* src, double* R)
{
    double rx = src[0], ry = src[1], rz = src[2];
    double theta = sqrt(rx * rx + ry * ry + rz * rz);
    for (int k = 0; k < 9; ++k) R[k] = (k % 4 == 0) ? 1.0 : 0.0;
    if (theta >= DBL_EPSILON) {
        double c, s; detSincos(theta, &s, &c);
        double c1 = 1. - c, it = theta ? 1. / theta : 0.;
        rx *= it; ry *= it; rz *= it;
        double rrt[9] = {rx * rx, rx * ry, rx * rz, rx * ry, ry * ry, ry * rz, rx * rz, ry * rz, rz * rz};
        double rxm[9] = {0, -rz, ry, rz, 0, -rx, -ry, rx, 0};
        for (int k = 0; k < 9; ++k) R[k] = c * ((k % 4 == 0) ? 1.0 : 0.0) + c1 * rrt[k] + s * rxm[k];
    }
}
__device__ void inv3d(const double* M, double* o)
{
    double c00 = M[4] * M[8] - M[5] * M[7], c01 = M[5] * M[6] - M[3] * M[8], c02 = M[3] * M[7] - M[4] * M[6];
    double det = M[0] * c00 + M[1] * c01 + M[2] * c02, id = 1.0 / det;
    o[0] = c00 * id; o[1] = (M[2] * M[7] - M[1] * M[8]) * id; o[2] = (M[1] * M[5] - M[2] * M[4]) * id;
    o[3] = c01 * id; o[4] = (M[0] * M[8] - M[2] * M[6]) * id; o[5] = (M[2] * M[3] - M[0] * M[5]) * id;
    o[6] = c02 * id; o[7] = (M[1] * M[6] - M[0] * M[7]) * id; o[8] = (M[0] * M[4] - M[1] * M[3]) * id;
}
__device__ void mul3d(const double* A, const double* B, double* C)
{
    double o[9];
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) o[r * 3 + c] = A[r * 3] * B[c] + A[r * 3 + 1] * B[3 + c] + A[r * 3 + 2] * B[6 + c];
    for (int k = 0; k < 9; ++k) C[k] = o[k];
}
__device__ void inv3f(const float* M, float* o)
{
    float c00 = M[4] * M[8] - M[5] * M[7], c01 = M[5] * M[6] - M[3] * M[8], c02 = M[3] * M[7] - M[4] * M[6];
    float det = (M[0] * c00 + M[1] * c01) + M[2] * c02, id = 1.0f / det;
    o[0] = c00 * id; o[1] = (M[2] * M[7] - M[1] * M[8]) * id; o[2] = (M[1] * M[5] - M[2] * M[4]) * id;
    o[3] = c01 * id; o[4] = (M[0] * M[8] - M[2] * M[6]) * id; o[5] = (M[2] * M[3] - M[0] * M[5]) * id;
    o[6] = c02 * id; o[7] = (M[1] * M[6] - M[0] * M[7]) * id; o[8] = (M[0] * M[4] - M[1] * M[3]) * id;
}

// per-level photometric constants: KRK^-1 and K t of the current estimate (RGBDOdometry.cpp:364-376)
__device__ void computeWarp(TrackState* st, Cam c)
{
    const double* T = st->resultRt;
    double R3[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]}, Ri[9], ti[3];
    inv3d(R3, Ri);
    for (int r = 0; r < 3; ++r) ti[r] = -(Ri[r * 3] * T[3] + Ri[r * 3 + 1] * T[7] + Ri[r * 3 + 2] * T[11]);
    double K[9] = {c.fx, 0, c.cx, 0, c.fy, c.cy, 0, 0, 1}, Kinv[9], tmp[9], KRK[9];
    inv3d(K, Kinv); mul3d(K, Ri, tmp); mul3d(tmp, Kinv, KRK);
    for (int q = 0; q < 9; ++q) st->krk[q] = (float)KRK[q];
    for (int r = 0; r < 3; ++r) st->kt[r] = (float)(K[r * 3] * ti[0] + K[r * 3 + 1] * ti[1] + K[r * 3 + 2] * ti[2]);
}

// ---------------------------------------------------------------------------------------
// block reduction helpers
// ---------------------------------------------------------------------------------------
template <int N>
MF_D void blockReduceStore(double* acc, double* partialOut)
{
    __shared__ double sh[TRK_THREADS / 32][N];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < N; ++k) {
        double v = acc[k];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) v += __hiloint2double(__shfl_down_sync(0xffffffffu, __double2hiint(v), off), __shfl_down_sync(0xffffffffu, __double2loint(v), off));
        if (lane == 0) sh[warp][k] = v;
    }
    __syncthreads();
    if (threadIdx.x < N) {
        double s = 0;
#pragma unroll
        for (int w = 0; w < TRK_THREADS / 32; ++w) s += sh[w][threadIdx.x];
        partialOut[threadIdx.x] = s;
    }
}

// Sum the per-block partials (rows of 32 doubles, N used) with the WHOLE last block: warp w takes blocks
// w, w+8, ...; lanes take columns lane and lane+32 (coalesced 128-byte rows, independent loads), doubles
// throughout; the 8 warp sums are combined in fixed order.  Deterministic for a fixed launch shape.
// (A single thread per column walking all partials serially exposes the L2 latency of every partial.)
template <int N>
MF_D void sumPartials(const double* __restrict__ partial, unsigned nblocks, double* tot /* shared, >= N */)
{
    __shared__ double ws[TRK_THREADS / 32][32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double a0 = 0;
#pragma unroll 4
    for (unsigned b = warp; b < nblocks; b += TRK_THREADS / 32) a0 += partial[(size_t)b * 32 + lane];
    ws[warp][lane] = a0;
    __syncthreads();
    if (threadIdx.x < N) {
        double s = 0;
#pragma unroll
        for (int w = 0; w < TRK_THREADS / 32; ++w) s += ws[w][threadIdx.x];
        tot[threadIdx.x] = s;
    }
    __syncthreads();
}

// returns true in ALL threads of the last block to arrive
MF_D bool lastBlock(unsigned* ticket)
{
    __shared__ bool isLast;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned t = atomicAdd(ticket, 1u);
        isLast = (t == gridDim.x - 1);
        if (isLast) *ticket = 0;
    }
    __syncthreads();
    if (isLast) __threadfence();
    return isLast;
}

// stand-alone ICP reduction at a caller-given pose (parity tests; mirrors icpStep's outputs)
__global__ void __launch_bounds__(TRK_THREADS) k_icp_only(const float4* __restrict__ vmapC, const float4* __restrict__ nmapC,
                                                          const float4* __restrict__ vmapG, const float4* __restrict__ nmapG,
                                                          int W, int H, Cam cam, TrackPoses pp, float distThres, float angleThres,
                                                          double* __restrict__ partial, unsigned* ticket, float* out29)
{
    // pp.p[0] = Rcurr(9) tcurr(3); pp.p[1] = RprevInv(9) tprev(3)
    double acc[NACC_ICP];
#pragma unroll
    for (int k = 0; k < NACC_ICP; ++k) acc[k] = 0.0;
    const float* Rc = pp.p[0]; const float* tc = pp.p[0] + 9; const float* Rpi = pp.p[1]; const float* tp = pp.p[1] + 9;
    const float3 tprev = make_float3(tp[0], tp[1], tp[2]);
    const int N = W * H;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < N; i += gridDim.x * blockDim.x) {
        float4 vc4 = vmapC[i];
        float3 vg = m3v(Rc, make_float3(vc4.x, vc4.y, vc4.z));
        vg = make_float3(vg.x + tc[0], vg.y + tc[1], vg.z + tc[2]);
        float3 vcp = m3v(Rpi, sub3(vg, tprev));
        int ux = __float2int_rn(vcp.x * cam.fx / vcp.z + cam.cx);
        int uy = __float2int_rn(vcp.y * cam.fy / vcp.z + cam.cy);
        if (ux < 0 || uy < 0 || ux >= W || uy >= H || vcp.z < 0) continue;
        int j = uy * W + ux;
        float4 vp4 = __ldg(vmapG + j), np4 = __ldg(nmapG + j), nc4 = nmapC[i];
        float3 vp = make_float3(vp4.x, vp4.y, vp4.z), np_ = make_float3(np4.x, np4.y, np4.z);
        float3 ng = m3v(Rc, make_float3(nc4.x, nc4.y, nc4.z));
        float3 d = sub3(vp, vg);
        float dist = sqrtf((d.x * d.x + d.y * d.y) + d.z * d.z);
        float3 c = cross3(ng, np_);
        float sine = sqrtf((c.x * c.x + c.y * c.y) + c.z * c.z);
        if (!(sine < angleThres && dist <= distThres && !isnan(nc4.x) && !isnan(np4.x))) continue;
        float3 s_cp = vcp, d_cp = m3v(Rpi, sub3(vp, tprev)), n_cp = m3v(Rpi, np_);
        float row[7];
        row[0] = n_cp.x; row[1] = n_cp.y; row[2] = n_cp.z;
        row[3] = s_cp.y * n_cp.z - s_cp.z * n_cp.y;
        row[4] = s_cp.z * n_cp.x - s_cp.x * n_cp.z;
        row[5] = s_cp.x * n_cp.y - s_cp.y * n_cp.x;
        row[6] = (n_cp.x * (s_cp.x - d_cp.x) + n_cp.y * (s_cp.y - d_cp.y)) + n_cp.z * (s_cp.z - d_cp.z);
        int q = 0;
#pragma unroll
        for (int a = 0; a < 6; ++a)
#pragma unroll
            for (int b = a; b < 7; ++b) { acc[q] = fma((double)row[a], (double)row[b], acc[q]); ++q; }
        acc[27] = fma((double)row[6], (double)row[6], acc[27]);
        acc[28] += 1.0;
    }
    blockReduceStore<NACC_ICP>(acc, partial + (size_t)blockIdx.x * 32);
    if (!lastBlock(ticket)) return;
    __shared__ double tot[NACC_ICP];
    sumPartials<NACC_ICP>(partial, gridDim.x, tot);
    if (threadIdx.x < NACC_ICP) out29[threadIdx.x] = (float)tot[threadIdx.x];
}

// =======================================================================================
// The whole Gauss-Newton schedule of a frame as ONE cooperative kernel.
//
// The reference returns to the host after each of its <= 67 reductions per model per frame; a launch-per-iteration
// device port pays launch + tail latency 38 times per frame.  Here a persistent grid (1 CTA per SM, CTA ranges per tracked model) walks the schedule
//     SO(3) pre-alignment (<= 10 its) -> level 2 (4) -> level 1 (5) -> level 0 (10)
// with one flagged exchange of partial rows per reduction.  The solver state is REPLICATED: after an exchange every CTA sums the
// same per-CTA partial rows in the same order and runs the same 6x6 solve, so all CTAs hold bit-identical poses and
// take identical break decisions without a second barrier or a broadcast.  Per-pixel data that a later phase needs
// (photometric correspondences, validity) is written and re-read by the same thread.
// =======================================================================================
#ifndef PT_THREADS
#define PT_THREADS 512
#endif
#define PT_WARPS (PT_THREADS / 32)
#define ROWF 32                        // doubles per partial row: two 128-byte lines per CTA per reduction

struct TrackParams {
    int W, H; Cam cam;
    int icp, rgb, rgbOnly, so3;
    int iterations[3];
    float icpWeight, angleThres, distThres, sobelScale, maxDepthDelta;
    float minScale[3];
    int corrSlots;                     // photometric correspondences kept per CTA in shared memory (0: global scratch instead)
    int bitWords;                      // shared-memory words reserved for the model-map validity bitmask of a level (0: none)
    int cacheRounds;                   // pixel rounds per thread whose pose-independent inputs are kept in shared memory across the iterations of a level
    unsigned llBase;                   // flag of the partial rows of reduction g of this launch: llBase + g (never 0)
    // flat grid: CTA b belongs to the job j with jobStart[j] <= b < jobStart[j + 1] -- the models of a batch get DIFFERENT numbers of
    // CTAs (a full-frame model walks 307 k live pixels per iteration, an object model rejects nearly all of them on its validity bitmask)
    int nJobs; unsigned short jobStart[TRACK_MAX_JOBS + 1];
};

// ---- per-warp normal equations on the fp64 tensor core ----
// A pixel contributes the outer product of its row (the Jacobian entries, the residual, and for ICP / SO(3) a 1 that counts it: 8 floats,
// zeros where unused) to an 8x8 sum.  One mma.m8n8k4.f64 (DMMA) adds 4 pixels: A = J^T (8 x 4), B = J (4 x 8), and lane l supplies the SAME
// value to both, component l >> 2 of pixel l & 3.  The accumulator fragment -- entries (l >> 2, 2 (l & 3)) and (l >> 2, 2 (l & 3) + 1) in
// lane l -- is the warp's sum over all its lanes: no per-thread accumulators across the pixel loop and no shuffle tree after it.  Every
// product of two floats is exact in fp64, so the sums are fp64 sums of exact products as before, in another order (R-SUM, DESIGN.md 4).
// A pixel's row goes straight to its lane's slot of a tile, so no row stays in registers while the other pixel in flight is worked on.
// A warp's two tiles share their shared memory with the fragment that the CTA reduction reads (the two are never live together).
union WarpScratch {
    float rows[2][32][8];              // rows of the two pixels in flight (lane l's in [.][l], read transposed by the MMAs)
    double frag[66];                   // the warp's 8x8 sum (row major) and its two integer counters
};

MF_D void putRow(float* slot, float4 lo, float4 hi)
{
    reinterpret_cast<float4*>(slot)[0] = lo;
    reinterpret_cast<float4*>(slot)[1] = hi;
}

// Adds the tile's rows to the warp's fragment f.  A lane whose row was not written (has = false) adds a zero row.  All 32 lanes must call.
MF_D void warpAccumulate(float (*tile)[8], bool has, double (&f)[2])
{
    if (!__any_sync(0xffffffffu, has)) return;             // 32 zero rows add +0.0 to sums that start at +0.0: skipping them is exact
    const int lane = threadIdx.x & 31;
    if (!has) putRow(tile[lane], make_float4(0.f, 0.f, 0.f, 0.f), make_float4(0.f, 0.f, 0.f, 0.f));
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const double v = (double)tile[4 * i + (lane & 3)][lane >> 2];   // lanes read 32 different banks
        asm("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};" : "+d"(f[0]), "+d"(f[1]) : "d"(v), "d"(v));
    }
    __syncwarp();                                          // the tile is rewritten by the next call
}

// Position in the 8x8 sum of accumulator q for rows of R entries (R - 1 Jacobian entries and the residual): q walks the upper triangle
// row by row without the residual's square (the layout solveAndUpdate and the SO(3) step read), then the residual's square, then the count.
template <int R>
MF_D int fragIndex(int q)
{
    constexpr int nJ = R * (R + 1) / 2 - 1;
    if (q == nJ) return (R - 1) * 9;
    if (q == nJ + 1) return R * 9;
    int a = 0;
    while (q >= R - a) { q -= R - a; ++a; }
    return a * 9 + q;
}

// ---- flagged exchange of the partial rows (the LL scheme of collective libraries) ----
// A row travels as 32 x 16 bytes {value.lo, flag, value.hi, flag}: every 8-byte half carries the flag of THIS reduction, 8-byte stores
// are single transactions, so a reader that finds both flags holds the value -- no release fence on the producer, no arrival counter,
// no second round trip for the data: the consumers poll the rows themselves.  The software barrier cost one fence + one atomic + one
// polled counter + one row read per reduction (48 reductions per frame); this costs the row read alone.
// Flags are unique per reduction and launch on one Model::partial buffer: llBase comes from the context's epoch (MaskFusion::trackEpoch),
// which advances by one per launch and skips the value whose llBase is 0, so a flag is never 0 -- the value of a fresh, zeroed buffer.
// Rows ping-pong between two buffers: a CTA writes reduction g + 2 only after it has consumed g + 1 from every peer, which every peer
// produced after consuming g.
MF_D void llStore(uint4* p, double v, unsigned flag)
{
    asm volatile("st.volatile.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"((unsigned)__double2loint(v)), "r"(flag), "r"((unsigned)__double2hiint(v)), "r"(flag) : "memory");
}
MF_D uint4 llLoad(const uint4* p)
{
    uint4 r;
    asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
    return r;
}

// CTA-wide fp64 sum of the warps' fragments -> one row of 32 flagged doubles in global memory (row = this CTA's partial): N (<= 29)
// accumulators, and two integer counters in columns 29 and 30 (exact in fp64).  Accumulating the exact products of floats in fp64 makes
// the totals agree with a sequential fp64 sum to ~1e-15 relative whatever the order: rounded to float (the reference's result record)
// they are the oracle's values bit for bit, which is what keeps tracked trajectories identical instead of merely close (DESIGN.md section 4).
// The warps' scratch is free again once every thread has passed the next barrier of sumRows.
template <int R, int N>
MF_D void ctaReduceStore(const double (&f)[2], WarpScratch* wsc, uint4* __restrict__ rowOut, unsigned flag, int extra0, int extra1)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int c0 = __reduce_add_sync(0xffffffffu, extra0), c1 = __reduce_add_sync(0xffffffffu, extra1);
    reinterpret_cast<double2*>(wsc[warp].frag)[lane] = make_double2(f[0], f[1]);
    if (lane == 0) { wsc[warp].frag[64] = (double)c0; wsc[warp].frag[65] = (double)c1; }
    __syncthreads();
    if (threadIdx.x < ROWF) {
        const int q = threadIdx.x;
        const int e = q < N ? fragIndex<R>(q) : (q == 29 || q == 30) ? 64 + (q - 29) : -1;
        double s = 0;
        if (e >= 0) {
#pragma unroll
            for (int w = 0; w < PT_WARPS; ++w) s += wsc[w].frag[e];
        }
        llStore(rowOut + q, s, flag);
    }
}
// every CTA: sum the R partial rows (fixed order, fp64) -> tot[0..32); columns 29/30 carry the integer counters.  Summation order:
// warp w adds rows w, w + 16, ... ascending, then the 16 warp sums are added ascending.  The rows of a batch are all polled until
// their flags match before the first add (one L2 round trip for R <= 160).
#define SUM_BATCH 10
MF_D void sumRows(const uint4* __restrict__ rows, unsigned R, unsigned flag, double (*ws)[ROWF], double* tot)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double a0 = 0;
    for (unsigned base = warp; base < R; base += PT_WARPS * SUM_BATCH) {
        uint4 x[SUM_BATCH];
        unsigned pending = 0;                                              // warp uniform: rows of the batch not yet seen complete
#pragma unroll
        for (int i = 0; i < SUM_BATCH; ++i) { x[i] = make_uint4(0, 0, 0, 0); if (base + (unsigned)i * PT_WARPS < R) pending |= 1u << i; }
        while (pending) {
#pragma unroll
            for (int i = 0; i < SUM_BATCH; ++i)
                if ((pending >> i) & 1u) x[i] = llLoad(rows + (size_t)(base + (unsigned)i * PT_WARPS) * ROWF + lane);
#pragma unroll
            for (int i = 0; i < SUM_BATCH; ++i)
                if ((pending >> i) & 1u) { if (__all_sync(0xffffffffu, x[i].y == flag && x[i].w == flag)) pending &= ~(1u << i); }
        }
#pragma unroll
        for (int i = 0; i < SUM_BATCH; ++i) a0 += __hiloint2double((int)x[i].z, (int)x[i].x);      // rows beyond R contribute +0.0
    }
    ws[warp][lane] = a0;
    __syncthreads();
    if (threadIdx.x < ROWF) {
        double s2 = 0;
#pragma unroll
        for (int w = 0; w < PT_WARPS; ++w) s2 += ws[w][threadIdx.x];
        tot[threadIdx.x] = s2;
    }
    __syncthreads();
}

// One reduction of the schedule: CTA partial -> flagged exchange -> every CTA holds the same totals (replicated solver state, no
// broadcast).  G CTAs of the model, the first Gact of them active.
struct RedCtx { uint4* rows; unsigned G, Gact, gen, llBase, bx; };
template <int R, int N>
MF_D void reduceStep(const double (&f)[2], int e0, int e1, bool active, RedCtx& rc, WarpScratch* wsc, double (*ws)[ROWF], double* tot)
{
    // 16 bytes per value: the two ping-pong buffers are G * ROWF values each
    uint4* rows = rc.rows + (size_t)(rc.gen & 1) * rc.G * ROWF;
    ++rc.gen;
    const unsigned flag = rc.llBase + rc.gen;
    if (active) ctaReduceStore<R, N>(f, wsc, rows + (size_t)rc.bx * ROWF, flag, e0, e1);
    sumRows(rows, rc.Gact, flag, ws, tot);
}

MF_D void gradU8(const uint8_t* __restrict__ img, int W, int x, int y, float& gx, float& gy)
{
    float actu = img[y * W + x], back = img[y * W + x - 1], fore = img[y * W + x + 1];
    gx = ((back + actu) / 2.0f) - ((fore + actu) / 2.0f);
    back = img[(y - 1) * W + x]; fore = img[(y + 1) * W + x];
    gy = ((back + actu) / 2.0f) - ((fore + actu) / 2.0f);
}


// entry e = (r, c) of the inverse of a 3x3: cofactor(c, r) / det with cyclic indices (no sign bookkeeping, no divergent
// switch: a 9-way switch serialised the nine lanes).  Products and differences are the ones inv3d forms.
// M is read in place with row stride LD (3 for a 3x3, 4 for the rotation block of a 4x4): no local copies.
template <int LD>
MF_D double inv3dEntry(const double* M, int e)
{
    const int r = e / 3, c = e - 3 * r;
    const int c1 = c == 2 ? 0 : c + 1, c2 = c1 == 2 ? 0 : c1 + 1, r1 = r == 2 ? 0 : r + 1, r2 = r1 == 2 ? 0 : r1 + 1;
    const double cof = M[c1 * LD + r1] * M[c2 * LD + r2] - M[c1 * LD + r2] * M[c2 * LD + r1];
    const double c00 = M[LD + 1] * M[2 * LD + 2] - M[LD + 2] * M[2 * LD + 1], c01 = M[LD + 2] * M[2 * LD] - M[LD] * M[2 * LD + 2],
                 c02 = M[LD] * M[2 * LD + 1] - M[LD + 1] * M[2 * LD];
    const double det = M[0] * c00 + M[1] * c01 + M[2] * c02;
    return cof * (1.0 / det);
}

// optional stage clock of the persistent kernel (A/B build -DMF_TRACK_TIMING; read back by mf_debug_track_timing): CTA 0 of model 0
// appends (tag, clock64) pairs at the stage boundaries of every reduction
#ifdef MF_TRACK_TIMING
__device__ long long g_trackTiming[8192];
__device__ int g_trackTimingN;
#define TT(tag) do { if (blockIdx.x == 0 && threadIdx.x == 0) { int q_ = g_trackTimingN; if (q_ + 2 <= 8192) { g_trackTiming[q_] = (tag); g_trackTiming[q_ + 1] = clock64(); g_trackTimingN = q_ + 2; } } } while (0)
#else
#define TT(tag) do { } while (0)
#endif

struct SolveScratch { double A[36], b[6], x[6], Rt[16], nr[16], Ri[9], K[9], Kinv[9], tmp[9], ti[3]; float trR[9], trT[3], iR[9], iT[3]; int fast; };

// computeWarp (RGBDOdometry.cpp:364-376) by one warp: every matrix entry keeps the scalar routine's formula, lanes take entries.
// sc->Kinv holds the inverse intrinsics of the level (set once per level).
MF_D void computeWarpCoop(TrackState* st, Cam c, SolveScratch* sc, int lane)
{
    const double* T = st->resultRt;
    const double* K = sc->K;
    if (lane < 9) sc->Ri[lane] = inv3dEntry<4>(T, lane);
    __syncwarp();
    if (lane < 3) sc->ti[lane] = -(sc->Ri[lane * 3] * T[3] + sc->Ri[lane * 3 + 1] * T[7] + sc->Ri[lane * 3 + 2] * T[11]);
    if (lane < 9) { int r = lane / 3, cc = lane % 3; sc->tmp[lane] = K[r * 3] * sc->Ri[cc] + K[r * 3 + 1] * sc->Ri[3 + cc] + K[r * 3 + 2] * sc->Ri[6 + cc]; }
    __syncwarp();
    if (lane < 9) { int r = lane / 3, cc = lane % 3; st->krk[lane] = (float)(sc->tmp[r * 3] * sc->Kinv[cc] + sc->tmp[r * 3 + 1] * sc->Kinv[3 + cc] + sc->tmp[r * 3 + 2] * sc->Kinv[6 + cc]); }
    if (lane < 3) st->kt[lane] = (float)(K[lane * 3] * sc->ti[0] + K[lane * 3 + 1] * sc->ti[1] + K[lane * 3 + 2] * sc->ti[2]);
    __syncwarp();
}

// host part of one Gauss-Newton iteration (RGBDOdometry.cpp:403-474) on the replicated state, executed by warp 0.
// Latency is all that matters here (every CTA runs the same solve while its other 15 warps wait), so the routine is laid out as four
// dependent stages instead of eleven: (1) every lane assembles ITS row of lastA / entry of lastb in registers straight from the totals and
// feeds the warp LDLT; (2) computeUpdateSE3: the scalar part in every lane, one entry of [R|t] per lane; (3) resultRt = Rt * resultRt;
// (4) everything derived from the new resultRt -- transform, its inverse, the current pose, and the photometric warp constants K R^-1 K^-1
// and K t -- is evaluated per output entry in registers (the 3x3 inverse redundantly in each lane: 50 fp64 operations cost less than
// the three shared-memory round trips they replace).  Every expression keeps the operand order of the staged version: same bits.
__device__ __noinline__ void solveAndUpdate(TrackState* st, const double* tot, bool ICP, bool RGB, float icpWeight, Cam cam, SolveScratch* sc)
{
    const int lane = threadIdx.x & 31;
    const double wgt = icpWeight;
    const int r6 = lane < 6 ? lane : 5;
    double arow[6], bown;
    {
        auto comb = [&](int c2, bool isA) -> double {
            const int a = r6 < c2 ? r6 : c2, b = r6 < c2 ? c2 : r6;
            const int q = 7 * a - (a * (a - 1)) / 2 + (b - a);
            const float vi = (float)tot[q], vr = (float)tot[NACC_ICP + q];
            if (ICP && RGB) return isA ? (double)vr + wgt * wgt * (double)vi : (double)vr + wgt * (double)vi;
            if (ICP) return (double)vi;
            return (double)vr;
        };
#pragma unroll
        for (int j = 0; j < 6; ++j) arow[j] = comb(j, true);
        bown = comb(6, false);
        if (lane < 6) {
#pragma unroll
            for (int j = 0; j < 6; ++j) st->lastA[lane * 6 + j] = arow[j];
            st->lastb[lane] = bown;
        }
    }
    if (ICP && lane == 31) { st->lastICPError = sqrtf((float)tot[27]) / (float)tot[28]; st->lastICPCount = (float)tot[28]; }
    TT(20);
    ldltSolvePivWarpRegs<6>(arow, bown, sc->x);
    TT(21);              // bit-identical to the sequential pivoted routine (Eigen's ldlt().solve conventions)
    // computeUpdateSE3 (OdometryProvider.h:69-90): Rt = [rodrigues(x[3..5]) | x[0..2]]; every lane evaluates the (cheap, identical)
    // scalar part, lanes < 16 assemble one entry each
    {
        double rx = sc->x[3], ry = sc->x[4], rz = sc->x[5];
        const double theta = sqrt(rx * rx + ry * ry + rz * rz);
        double c = 1.0, s = 0.0, c1 = 0.0;
        const bool rot = theta >= DBL_EPSILON;
        if (rot) { detSincos(theta, &s, &c); c1 = 1. - c; const double it = 1. / theta; rx *= it; ry *= it; rz *= it; }
        if (lane < 16) {
            const int r = lane >> 2, cc = lane & 3;
            double v;
            if (r == 3) v = cc == 3 ? 1.0 : 0.0;
            else if (cc == 3) v = sc->x[r];
            else if (!rot) v = r == cc ? 1.0 : 0.0;
            else {
                const double ur = r == 0 ? rx : r == 1 ? ry : rz, uc = cc == 0 ? rx : cc == 1 ? ry : rz;
                const double rrt = ur * uc;
                // [r]_x entries: (0,1) -rz (0,2) ry (1,0) rz (1,2) -rx (2,0) -ry (2,1) rx
                const int d = cc - r;                                  // +-1, +-2
                const int o = 3 - r - cc;                              // the third index
                const double uo = o == 0 ? rx : o == 1 ? ry : rz;
                const double rxm = (r == cc) ? 0.0 : ((d == 1 || d == -2) ? -uo : uo);
                v = c * (r == cc ? 1.0 : 0.0) + c1 * rrt + s * rxm;
            }
            sc->Rt[lane] = v;
        }
    }
    __syncwarp();
    TT(22);
    if (lane < 16) {
        const int r = lane >> 2, c = lane & 3;
        double s2 = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) s2 += sc->Rt[r * 4 + k] * st->resultRt[k * 4 + c];
        sc->nr[lane] = s2;                                 // the new resultRt (st->resultRt is still being read by the other lanes)
    }
    __syncwarp();
    // ---- stage 4: every output entry from nr[] in registers ----
    const double* T = sc->nr;
    if (lane < 16) st->resultRt[lane] = T[lane];
    // transform (float) = [trR | trT]; currentT = [Rprev|tprev] * transform^-1 (RGBDOdometry.cpp:466-474): iR = trR^T, iT = -iR trT
    if (lane < 9) st->trR[lane] = (float)T[(lane / 3) * 4 + lane % 3];
    else if (lane < 12) st->trT[lane - 9] = (float)T[(lane - 9) * 4 + 3];
    if (lane < 9) {
        const int r = lane / 3, c = lane % 3;
        // iR[k][c] = trR[c][k]
        const float i0 = (float)T[c * 4 + 0], i1 = (float)T[c * 4 + 1], i2 = (float)T[c * 4 + 2];
        st->Rcurr[lane] = (st->Rprev[r * 3] * i0 + st->Rprev[r * 3 + 1] * i1) + st->Rprev[r * 3 + 2] * i2;
    } else if (lane < 12) {
        const int r = lane - 9;
        const float t0 = (float)T[3], t1 = (float)T[7], t2 = (float)T[11];
        float iT[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) iT[k] = -(((float)T[0 * 4 + k] * t0 + (float)T[1 * 4 + k] * t1) + (float)T[2 * 4 + k] * t2);
        st->tcurr[r] = ((st->Rprev[r * 3] * iT[0] + st->Rprev[r * 3 + 1] * iT[1]) + st->Rprev[r * 3 + 2] * iT[2]) + st->tprev[r];
    }
    TT(23);
    if (RGB && lane >= 16 && lane < 28) {
        // computeWarp (RGBDOdometry.cpp:364-376): K R^-1 K^-1 and K t^-1 of the new estimate for the next iteration's residuals; lanes 16..24
        // take one entry of KRK^-1 each, lanes 25..27 one entry of Kt (the lanes that are idle in the float part above)
        const double* K = sc->K;
        double Ri[9];
#pragma unroll
        for (int e = 0; e < 9; ++e) Ri[e] = inv3dEntry<4>(T, e);
        const int l = lane - 16;
        if (l < 9) {
            const int r = l / 3, cc = l % 3;
            double tmp[3];
#pragma unroll
            for (int j = 0; j < 3; ++j) tmp[j] = K[r * 3] * Ri[j] + K[r * 3 + 1] * Ri[3 + j] + K[r * 3 + 2] * Ri[6 + j];
            st->krk[l] = (float)(tmp[0] * sc->Kinv[cc] + tmp[1] * sc->Kinv[3 + cc] + tmp[2] * sc->Kinv[6 + cc]);
        } else {
            const int q = l - 9;
            double ti[3];
#pragma unroll
            for (int j = 0; j < 3; ++j) ti[j] = -(Ri[j * 3] * T[3] + Ri[j * 3 + 1] * T[7] + Ri[j * 3 + 2] * T[11]);
            st->kt[q] = (float)(K[q * 3] * ti[0] + K[q * 3 + 1] * ti[1] + K[q * 3 + 2] * ti[2]);
        }
    }
}

MF_D void prefetchL1(const void* p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }

// one pixel of phase A through its four stages; two of these are in flight per thread (their gathers overlap)
struct PixA {
    float4 vc, nc; float d1; int valid, ni, x, y;                 // pose-independent inputs
    bool rOK, iOK; int jr, ji, u0, v0; float td1; float3 vg, vcp;  // projections under the current estimate
    float d0; int li; float4 vp4, np4;                             // gathered model data
};

extern __shared__ int2 corrShared[];

// the whole schedule of a frame for every tracked model: cooperative launch, one CTA per SM
__global__ void __launch_bounds__(PT_THREADS, 1) k_track_persistent(const TrackJob* __restrict__ jobs, TrackParams tp)
{
    __shared__ TrackJob J;
    __shared__ TrackState S;
    __shared__ SolveScratch sc;
    __shared__ __align__(16) WarpScratch wsc[PT_WARPS];
    __shared__ double ws[PT_WARPS][ROWF];
    __shared__ double tot[64];
    __shared__ double totR[ROWF];
    __shared__ float so3B[9], so3Kinv[9], so3Krlr[9];
    __shared__ double so3K[9], so3KinvD[9];
    __shared__ int flag;
    unsigned job = 0;                                                  // the model of this CTA
    while ((int)job + 1 < tp.nJobs && blockIdx.x >= tp.jobStart[job + 1]) ++job;
    const unsigned bx = blockIdx.x - tp.jobStart[job];                 // CTA index within its model
    const unsigned G = (unsigned)tp.jobStart[job + 1] - tp.jobStart[job];      // CTAs of this model
    {   // job record -> shared memory (one coalesced read instead of dependent pointer chases in every phase)
        const uint32_t* src = reinterpret_cast<const uint32_t*>(jobs + job);
        uint32_t* dst = reinterpret_cast<uint32_t*>(&J);
        for (int k = threadIdx.x; k < (int)(sizeof(TrackJob) / 4); k += PT_THREADS) dst[k] = src[k];
    }
    TrackState* st = &S;
#ifdef MF_TRACK_TIMING
    if (blockIdx.x == 0 && threadIdx.x == 0) g_trackTimingN = 0;
#endif
    TT(1);
    __syncthreads();
    if (threadIdx.x == 0) {
        // RGBDOdometry.cpp:331-345 initial state; the model's pose is device resident (written by the previous frame's epilogue or k_set_pose)
        const float* P = J.dpose->pose.m;
        for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) st->Rprev[r * 3 + c] = P[r * 4 + c]; st->tprev[r] = P[r * 4 + 3]; }
        for (int k = 0; k < 9; ++k) st->Rcurr[k] = st->Rprev[k];
        for (int k = 0; k < 3; ++k) st->tcurr[k] = st->tprev[k];
        inv3f(st->Rprev, st->RprevInv);
        for (int k = 0; k < 16; ++k) st->resultRt[k] = (k % 5 == 0) ? 1.0 : 0.0;
        for (int k = 0; k < 9; ++k) { st->resultR[k] = (k % 4 == 0) ? 1.0 : 0.0; st->lastResultR[k] = st->resultR[k]; st->R_lr[k] = (k % 4 == 0) ? 1.f : 0.f; st->trR[k] = (k % 4 == 0) ? 1.f : 0.f; }
        st->trT[0] = st->trT[1] = st->trT[2] = 0;
        st->so3LastError = FLT_MAX / 2; st->so3LastCount = FLT_MAX / 2; st->so3Done = 0;
        st->levelBreak = 0; st->lastRGBError = FLT_MAX; st->lastRGBCount = 0; st->lastICPError = 0; st->lastICPCount = 0;
        st->lastSO3Error = 0; st->lastSO3Count = 0; st->sigmaVal = 0;
        for (int k = 0; k < 36; ++k) st->lastA[k] = 0;
        for (int k = 0; k < 6; ++k) st->lastb[k] = 0;
    }
    __syncthreads();
    RedCtx rc;
    rc.rows = reinterpret_cast<uint4*>(J.partial); rc.G = G; rc.Gact = G; rc.gen = 0; rc.llBase = tp.llBase; rc.bx = bx;
    // photometric correspondences of this thread's pixels, slot = round * PT_THREADS + thread: written in phase A, read in phase B
    // by the same thread.  Shared memory when the launch reserved enough, else a private stripe of the model's scratch buffer.
    const size_t corrNeed = (size_t)((tp.W * tp.H + G * PT_THREADS - 1) / (G * PT_THREADS)) * PT_THREADS;      // slots of this CTA at level 0 (depends on the model's share of the grid)
    int2* const corr = ((size_t)tp.corrSlots >= corrNeed && tp.corrSlots) ? corrShared : reinterpret_cast<int2*>(J.corres[0]) + (size_t)bx * corrNeed;
    // Pose-independent inputs of this thread's pixels (frame vertex / normal, depth of the photometric pyramid, intensity, validity, image
    // gradient, pixel coordinates) are the same in every iteration of a level: they are read from global memory ONCE per level into
    // shared memory (slot = round * PT_THREADS + thread, structure of arrays: conflict-free 16-byte accesses) and the Gauss-Newton
    // iterations re-read them from there.  Phase A then issues only its pose-dependent gathers: one L2 round trip instead of two, fewer
    // instructions per pixel.  Rounds beyond tp.cacheRounds (720p level 0) use global memory.
    const int cacheSlots = tp.cacheRounds * PT_THREADS;
    unsigned char* const cacheBase = reinterpret_cast<unsigned char*>(corrShared) + (((size_t)tp.corrSlots * sizeof(int2) + 15) & ~(size_t)15);
    float4* const vcS = reinterpret_cast<float4*>(cacheBase);
    float4* const ncS = vcS + cacheSlots;
    float* const d1S = reinterpret_cast<float*>(ncS + cacheSlots);
    uint32_t* const pkS = reinterpret_cast<uint32_t*>(d1S + cacheSlots);          // valid | intensity << 1 | x << 9 | y << 20
    uint32_t* const gS = pkS + cacheSlots;                                         // Sobel gradient (short2 bits)
    uint32_t* const bitsS = gS + cacheSlots;                                       // validity bitmask of the model's normal map at this level

    // ---------------- SO(3) pre-alignment on level-2 intensities (RGBDOdometry.cpp:272-345) ----------------
    if (tp.so3) {
        const int W = tp.W >> 2, H = tp.H >> 2, N = W * H;
        // CTAs beyond the pixel count only wait at the barriers: fewer partial rows to sum
        const unsigned Gact = min(G, (unsigned)((N + PT_THREADS - 1) / PT_THREADS));
        const bool active = bx < Gact;
        const int tid = (int)bx * PT_THREADS + threadIdx.x, nthr = (int)Gact * PT_THREADS;
        const Cam c = camLevel(tp.cam, 2);
        const uint8_t* __restrict__ lastImage = J.lastNextImage2;
        const uint8_t* __restrict__ nextImage = J.nextImage[2];
        if (threadIdx.x == 0) {
            double K[9] = {c.fx, 0, c.cx, 0, c.fy, c.cy, 0, 0, 1}, Kinv[9];
            inv3d(K, Kinv);
            for (int q = 0; q < 9; ++q) { so3K[q] = K[q]; so3KinvD[q] = Kinv[q]; so3Kinv[q] = (float)Kinv[q]; }
        }
        __syncthreads();
        for (int it = 0; it < 10; ++it) {
            if (threadIdx.x < 9) {
                // homography K R K^-1 of the current estimate, one entry per lane (same sums as mul3d)
                const int r = threadIdx.x / 3, cc = threadIdx.x % 3;
                double kr[3];
#pragma unroll
                for (int q = 0; q < 3; ++q) kr[q] = so3K[r * 3] * st->resultR[q] + so3K[r * 3 + 1] * st->resultR[3 + q] + so3K[r * 3 + 2] * st->resultR[6 + q];
                so3Krlr[threadIdx.x] = (float)(cc == 0 ? kr[0] : cc == 1 ? kr[1] : kr[2]);     // constant indices: kr[] stays in registers
                so3B[threadIdx.x] = (float)(kr[0] * so3KinvD[cc] + kr[1] * so3KinvD[3 + cc] + kr[2] * so3KinvD[6 + cc]);
            }
            __syncthreads();
            TT(11);
            double f[2] = {0.0, 0.0};
            if (active) {
                // warp-uniform trip count (the MMAs need all 32 lanes): a lane past the last pixel adds a zero row
                for (int k0 = tid - (threadIdx.x & 31); k0 < N; k0 += nthr) {
                    const int k = k0 + (threadIdx.x & 31);
                    int y = k / W, x = k - y * W;
                    float3 ur = make_float3((float)x, (float)y, 1.0f);
                    float3 wr = m3v(so3B, ur);
                    int wx = __float2int_rn(wr.x / wr.z), wy = __float2int_rn(wr.y / wr.z);
                    bool found = (k < N && wx >= 1 && wx < W - 1 && wy >= 1 && wy < H - 1 && x >= 1 && x < W - 1 && y >= 1 && y < H - 1);
                    if (found) {
                        float gnx, gny, glx, gly;
                        gradU8(nextImage, W, wx, wy, gnx, gny);
                        gradU8(lastImage, W, x, y, glx, gly);
                        float gx = (gnx + glx) / 2.0f, gy = (gny + gly) / 2.0f;
                        float3 p = m3v(so3Kinv, ur);
                        float z2 = p.z * p.z;
                        float a = so3Krlr[0], b = so3Krlr[1], cc = so3Krlr[2], d = so3Krlr[3], e = so3Krlr[4], f = so3Krlr[5], g = so3Krlr[6], h = so3Krlr[7], i = so3Krlr[8];
                        float fy = (float)y, fxx = (float)x;
                        float3 l = make_float3(((p.z * (d * gy + a * gx)) - (gy * g * fy) - (gx * g * fxx)) / z2,
                                               ((p.z * (e * gy + b * gx)) - (gy * h * fy) - (gx * h * fxx)) / z2,
                                               ((p.z * (f * gy + cc * gx)) - (gy * i * fy) - (gx * i * fxx)) / z2);
                        // column 4 counts the pixel
                        putRow(wsc[threadIdx.x >> 5].rows[0][threadIdx.x & 31],
                               make_float4(l.y * p.z - l.z * p.y, l.z * p.x - l.x * p.z, l.x * p.y - l.y * p.x, -((float)nextImage[wy * W + wx] - (float)lastImage[k])),
                               make_float4(1.f, 0.f, 0.f, 0.f));
                    }
                    warpAccumulate(wsc[threadIdx.x >> 5].rows[0], found, f);
                }
            }
            TT(12);
            rc.Gact = Gact;
            reduceStep<4, 11>(f, 0, 0, active, rc, wsc, ws, tot);
            TT(15);
            if (threadIdx.x < 32) {
                // host logic of RGBDOdometry.cpp:301-324 on warp 0: lane 0 takes the decisions, the 3x3 solve is warp-cooperative
                int mode = 0;                                  // 0: converged, 1: diverged (restore), 2: step
                if (threadIdx.x == 0) {
                    float res0 = (float)tot[9], res1 = (float)tot[10];
                    st->lastSO3Error = sqrtf(res0) / res1; st->lastSO3Count = res1;
                    if (st->lastSO3Error < st->so3LastError && fabsf(st->so3LastError - st->lastSO3Count) < 0.001f) mode = 0;
                    else if (st->lastSO3Error > st->so3LastError + 0.001f) {
                        st->lastSO3Error = st->so3LastError; st->lastSO3Count = st->so3LastCount;
                        for (int q = 0; q < 9; ++q) st->resultR[q] = st->lastResultR[q];
                        mode = 1;
                    } else {
                        st->so3LastError = st->lastSO3Error; st->so3LastCount = st->lastSO3Count;
                        for (int q = 0; q < 9; ++q) st->lastResultR[q] = st->resultR[q];
                        double* A = sc.A; double* bb = sc.b;
                        A[0] = (double)(float)tot[0]; A[1] = A[3] = (double)(float)tot[1]; A[2] = A[6] = (double)(float)tot[2]; bb[0] = (double)(float)tot[3];
                        A[4] = (double)(float)tot[4]; A[5] = A[7] = (double)(float)tot[5]; bb[1] = (double)(float)tot[6];
                        A[8] = (double)(float)tot[7]; bb[2] = (double)(float)tot[8];
                        mode = 2;
                    }
                }
                mode = __shfl_sync(0xffffffffu, mode, 0);
                if (mode == 2) {
                    __syncwarp();
                    ldltSolvePivWarp<3>(sc.A, sc.b, sc.x);
                    if (threadIdx.x == 0) {
                        double delta[3];
                        for (int k = 0; k < 3; ++k) delta[k] = (double)(float)sc.x[k];
                        double ru[9]; rodrigues(delta, ru);
                        float ruf[9], n[9];
                        for (int k = 0; k < 9; ++k) ruf[k] = (float)ru[k];
                        for (int r = 0; r < 3; ++r) for (int cc2 = 0; cc2 < 3; ++cc2) n[r * 3 + cc2] = (ruf[r * 3] * st->R_lr[cc2] + ruf[r * 3 + 1] * st->R_lr[3 + cc2]) + ruf[r * 3 + 2] * st->R_lr[6 + cc2];
                        for (int k = 0; k < 9; ++k) { st->R_lr[k] = n[k]; st->resultR[k] = n[k]; }
                    }
                }
                if (threadIdx.x == 0) flag = mode != 2;
            }
            TT(16);
            __syncthreads();
            if (flag) break;
        }
        __syncthreads();
        if (threadIdx.x == 0)          // so3 result -> initial resultRt (RGBDOdometry.cpp:337-345)
            for (int r = 0; r < 3; ++r) for (int cc = 0; cc < 3; ++cc) st->resultRt[r * 4 + cc] = st->resultR[r * 3 + cc];
        __syncthreads();
    }

    // ---------------- pyramid levels, coarse to fine (RGBDOdometry.cpp:347-476) ----------------
    for (int level = 2; level >= 0; --level) {
        if (tp.iterations[level] == 0) continue;
        const int W = tp.W >> level, H = tp.H >> level, N = W * H;
        const unsigned Gact = min(G, (unsigned)((N + PT_THREADS - 1) / PT_THREADS));
        const bool active = bx < Gact;
        const int tid = (int)bx * PT_THREADS + threadIdx.x, nthr = (int)Gact * PT_THREADS;
        // Pixels of this thread: tid + r * nthr for the fullRounds rounds every thread has, plus at most one pixel of the tail
        // (N - fullRounds * nthr pixels).  The tail is dealt out by warps of 32 pixels ACROSS the CTAs (tail warp j -> CTA j % Gact,
        // warp j / Gact): at 640x480 on 148 CTAs the 4096 tail pixels become one extra pixel for ONE warp of 128 CTAs instead of a
        // fifth round (= a third pair of the two-deep pipeline below) for ALL warps of CTAs 0..7, which every other CTA then waited
        // for at the grid barrier of each of the ten iterations.
        const int fullRounds = N / nthr;
        int kTail = -1;
        if (active) {
            const int j = (threadIdx.x >> 5) * (int)Gact + (int)bx;
            const int kt = fullRounds * nthr + j * 32 + (threadIdx.x & 31);
            if (kt < N) kTail = kt;
        }
        const int rounds = active ? fullRounds + (kTail >= 0 ? 1 : 0) : 0;
        // rounds of the warp (the MMAs need all 32 lanes): a lane without a pixel in the last one adds zero rows
        const bool tailW = __any_sync(0xffffffffu, kTail >= 0);
        const int roundsW = active ? fullRounds + (tailW ? 1 : 0) : 0;
        auto kOf = [&](int r) { return r < fullRounds ? tid + r * nthr : kTail; };
        float (*const tiles)[32][8] = wsc[threadIdx.x >> 5].rows;
        const Cam cam = camLevel(tp.cam, level);
        const float4* __restrict__ vmapC = J.vmapC[level];
        const float4* __restrict__ nmapC = J.nmapC[level];
        const float4* __restrict__ vmapG = J.vmapG[level];
        const float4* __restrict__ nmapG = J.nmapG[level];
        const float4* __restrict__ cloud = J.cloud[level];
        const short2* __restrict__ grad = J.nextGrad[level];
        const float* __restrict__ lastDepth = J.lastDepth[level];
        const float* __restrict__ nextDepth = J.lastDepth[level];      // reference quirk: both pyramids derive from vmaps_tmp (RGBDOdometry.cpp:187-215)
        const uint8_t* __restrict__ lastImage = J.lastImage[level];
        const uint8_t* __restrict__ nextImage = J.nextImage[level];
        const uint8_t* __restrict__ rgbValid = J.rgbValid[level];         // pose-independent validity, written by k_sobel
        if (threadIdx.x < 32) {
            if (threadIdx.x == 0) { st->levelBreak = 0; st->lastRGBError = FLT_MAX; }
            if (threadIdx.x < 9) {
                const int r = threadIdx.x / 3, cc = threadIdx.x % 3;
                sc.K[threadIdx.x] = r == cc ? (r == 0 ? (double)cam.fx : r == 1 ? (double)cam.fy : 1.0) : (cc == 2 ? (r == 0 ? (double)cam.cx : (double)cam.cy) : 0.0);
            }
            __syncwarp();
            if (threadIdx.x < 9) sc.Kinv[threadIdx.x] = inv3dEntry<3>(sc.K, threadIdx.x);
            __syncwarp();
            if (tp.rgb) computeWarpCoop(st, cam, &sc, threadIdx.x);
        }
        __syncthreads();

        // object models: validity bitmask of this level's model maps -> shared memory (every CTA holds the whole level: gathers go anywhere)
        const bool useBits = tp.icp && tp.bitWords > 0 && J.validBits[level] != nullptr && (N + 31) / 32 <= tp.bitWords;
        if (useBits) {
            const uint32_t* __restrict__ src = J.validBits[level];
            for (int k = threadIdx.x; k < (N + 31) / 32; k += PT_THREADS) bitsS[k] = __ldg(src + k);
        }
        __syncthreads();
        // fill the per-level cache (see cacheSlots above)
        const int cRounds = min(rounds, tp.cacheRounds);
        for (int r = 0; r < cRounds; ++r) {
            const int k = kOf(r), slot = r * PT_THREADS + threadIdx.x;
            const int y = k / W, x = k - y * W;
            uint32_t pk = ((uint32_t)x << 9) | ((uint32_t)y << 20);
            float d1 = 0.f; float4 vc = make_float4(0, 0, 0, 0), nc = vc; uint32_t g = 0;
            if (tp.rgb) { pk |= (rgbValid[k] ? 1u : 0u) | ((uint32_t)nextImage[k] << 1); d1 = nextDepth[k]; const short2 gg = grad[k]; g = (uint32_t)(uint16_t)gg.x | ((uint32_t)(uint16_t)gg.y << 16); }
            if (tp.icp) { vc = vmapC[k]; nc = nmapC[k]; }
            vcS[slot] = vc; ncS[slot] = nc; d1S[slot] = d1; pkS[slot] = pk; gS[slot] = g;
        }
        // pose-independent inputs of pixel k (round r)
        auto stage0 = [&](PixA& p, int k, int r) {
            if (r < cRounds) {
                const int slot = r * PT_THREADS + threadIdx.x;
                const uint32_t pk = pkS[slot];
                p.valid = (int)(pk & 1u); p.ni = (int)((pk >> 1) & 0xffu); p.x = (int)((pk >> 9) & 0x7ffu); p.y = (int)(pk >> 20);
                p.d1 = d1S[slot]; p.vc = vcS[slot]; p.nc = ncS[slot];
                return;
            }
            p.valid = 0; p.d1 = 0.f; p.ni = 0; p.vc = make_float4(0, 0, 0, 0); p.nc = p.vc;
            p.y = k / W; p.x = k - p.y * W;
            if (tp.rgb) { p.valid = rgbValid[k]; p.d1 = nextDepth[k]; p.ni = nextImage[k]; }
            if (tp.icp) { p.vc = vmapC[k]; p.nc = nmapC[k]; }
        };
        auto noPixel0 = [&](PixA& p) { p.valid = 0; p.d1 = 0.f; p.ni = 0; p.x = 0; p.y = 0; p.vc = make_float4(0, 0, 0, 0); p.nc = p.vc; };
        // (Tried: source pixels whose model-side depth is exactly 0 -- 95 % of an object model's image -- all warp to ONE target pixel, so
        // whether they can correspond is decidable once per iteration and they could skip the photometric projection.  Exact, but the two
        // dependent loads of that decision sat on the critical path of every iteration and made the
        // tracker slower.  Removed.)
        // addresses of both gathers under the current estimate
        auto stage1 = [&](PixA& p, int k, const float3 tprev) {
            p.rOK = false; p.iOK = false; p.jr = 0; p.ji = 0; p.u0 = 0; p.v0 = 0; p.td1 = 0.f;
            p.vg = make_float3(0, 0, 0); p.vcp = p.vg;
            const int y = p.y, x = p.x;
            if (tp.rgb && p.valid && !isnan(p.d1)) {
                const float* K = st->krk; const float* kt = st->kt;
                const float d1 = p.d1;
                p.td1 = d1 * ((K[6] * x + K[7] * y) + K[8]) + kt[2];
                float fu = (d1 * ((K[0] * x + K[1] * y) + K[2]) + kt[0]) / p.td1;
                float fv = (d1 * ((K[3] * x + K[4] * y) + K[5]) + kt[1]) / p.td1;
                p.u0 = (fu != fu || fabsf(fu) > 1e9f) ? -1 : __float2int_rn(fu);
                p.v0 = (fv != fv || fabsf(fv) > 1e9f) ? -1 : __float2int_rn(fv);
                if (p.u0 >= 0 && p.v0 >= 0 && p.u0 < W && p.v0 < H) { p.rOK = true; p.jr = p.v0 * W + p.u0; }
            }
            if (tp.icp) {
                float3 vg = m3v(st->Rcurr, make_float3(p.vc.x, p.vc.y, p.vc.z));
                vg = make_float3(vg.x + st->tcurr[0], vg.y + st->tcurr[1], vg.z + st->tcurr[2]);
                float3 vcp = m3v(st->RprevInv, sub3(vg, tprev));
                int ux = __float2int_rn(vcp.x * cam.fx / vcp.z + cam.cx);
                int uy = __float2int_rn(vcp.y * cam.fy / vcp.z + cam.cy);
                if (!(ux < 0 || uy < 0 || ux >= W || uy >= H || vcp.z < 0)) {
                    p.ji = uy * W + ux;
                    // the correspondence needs a valid model normal at ji (reduce.cu:346-352): known from the bitmask without the gathers
                    p.iOK = !useBits || ((bitsS[p.ji >> 5] >> (p.ji & 31)) & 1u);
                }
                p.vg = vg; p.vcp = vcp;
            }
        };
        auto noPixel1 = [&](PixA& p) { p.rOK = false; p.iOK = false; p.jr = 0; p.ji = 0; p.u0 = 0; p.v0 = 0; p.td1 = 0.f; p.vg = make_float3(0, 0, 0); p.vcp = p.vg; };
        auto stage2 = [&](PixA& p) {
            p.d0 = 0.f; p.li = 0; p.vp4 = make_float4(0, 0, 0, 0); p.np4 = p.vp4;
            if (p.rOK) { p.d0 = lastDepth[p.jr]; p.li = lastImage[p.jr]; }
            if (p.iOK) { p.vp4 = __ldg(vmapG + p.ji); p.np4 = __ldg(nmapG + p.ji); }
        };

        for (int it = 0; it < tp.iterations[level]; ++it) {
            // ---- phase A: photometric correspondences + statistics, ICP normal equations ----
            TT(100 + level);
            double f[2] = {0.0, 0.0};
            int cnt = 0, sig = 0;
            if (active) {
                const float3 tprev = make_float3(st->tprev[0], st->tprev[1], st->tprev[2]);
                // arithmetic of one pixel: photometric correspondence and statistics; returns whether it is an ICP correspondence, whose
                // row (and a 1 that counts it) goes to `row`
                auto stage3 = [&](const PixA& p, int slot, float* row) -> bool {
                    if (tp.rgb) {
                        int2 c = make_int2(-1, 0);                     // .x = u0 | v0 << 16 (or -1: no correspondence), .y = bits of diff
                        if (p.rOK && p.d0 > 0 && fabsf(p.td1 - p.d0) <= tp.maxDepthDelta && p.li != 0) {
                            const float diff = (float)p.ni - (float)p.li;
                            c.x = (p.u0 & 0xffff) | (p.v0 << 16); c.y = __float_as_int(diff);
                            cnt += 1;
                            sig += (int)(diff * diff);
                        }
                        corr[slot] = c;
                    }
                    if (p.iOK) {
                        const float4 nc4 = p.nc, vp4 = p.vp4, np4 = p.np4;
                        float3 vp = make_float3(vp4.x, vp4.y, vp4.z), np_ = make_float3(np4.x, np4.y, np4.z);
                        float3 ng = m3v(st->Rcurr, make_float3(nc4.x, nc4.y, nc4.z));
                        float3 d = sub3(vp, p.vg);
                        float dist = sqrtf((d.x * d.x + d.y * d.y) + d.z * d.z);
                        float3 c = cross3(ng, np_);
                        float sine = sqrtf((c.x * c.x + c.y * c.y) + c.z * c.z);
                        bool found = (sine < tp.angleThres && dist <= tp.distThres && !isnan(nc4.x) && !isnan(np4.x));
                        if (found) {
                            float3 s_cp = p.vcp;
                            float3 d_cp = m3v(st->RprevInv, sub3(vp, tprev));
                            float3 n_cp = m3v(st->RprevInv, np_);
                            putRow(row, make_float4(n_cp.x, n_cp.y, n_cp.z, s_cp.y * n_cp.z - s_cp.z * n_cp.y),
                                   make_float4(s_cp.z * n_cp.x - s_cp.x * n_cp.z, s_cp.x * n_cp.y - s_cp.y * n_cp.x,
                                               (n_cp.x * (s_cp.x - d_cp.x) + n_cp.y * (s_cp.y - d_cp.y)) + n_cp.z * (s_cp.z - d_cp.z), 1.f));
                            return true;
                        }
                    }
                    return false;
                };
                for (int r = 0; r < roundsW; r += 2) {
                    const bool hasA = r < rounds, hasB = r + 1 < rounds;
                    const int k0 = hasA ? kOf(r) : 0, k1 = hasB ? kOf(r + 1) : k0;
                    // next pair's streaming inputs -> L1 while this pair's dependent gathers are in flight (rounds not held in shared memory)
                    for (int q = 2; q < 4; ++q)
                        if (r + q < rounds && r + q >= cRounds) {
                            const int kn = kOf(r + q);
                            if (tp.icp) { prefetchL1(vmapC + kn); prefetchL1(nmapC + kn); }
                            if (tp.rgb) { prefetchL1(nextDepth + kn); }
                        }
                    PixA a, b;
                    if (hasA) stage0(a, k0, r); else noPixel0(a);
                    if (hasB) stage0(b, k1, r + 1); else noPixel0(b);
                    if (hasA) stage1(a, k0, tprev); else noPixel1(a);
                    if (hasB) stage1(b, k1, tprev); else noPixel1(b);
                    stage2(a); stage2(b);
                    const bool fA = hasA && stage3(a, r * PT_THREADS + threadIdx.x, tiles[0][threadIdx.x & 31]);
                    const bool fB = hasB && stage3(b, (r + 1) * PT_THREADS + threadIdx.x, tiles[1][threadIdx.x & 31]);
                    warpAccumulate(tiles[0], fA, f);
                    warpAccumulate(tiles[1], fB, f);
                }
            }
            TT(2);
            rc.Gact = Gact;
            // phase B's first streaming inputs (pose independent) -> L1 while this CTA waits at the reduction
            if (tp.rgb && rounds > cRounds) { prefetchL1(grad + kOf(cRounds)); }
            reduceStep<7, NACC_ICP>(f, cnt, sig, active, rc, wsc, ws, tot);
            TT(5);
            if (tp.rgb) {
                if (threadIdx.x == 0) {
                    // RGBDOdometry.cpp:388-401
                    int rgbSize = (int)(long long)tot[29], sigma = (int)(long long)tot[30];
                    float tmpError = (float)(sqrt((double)sigma) / (double)rgbSize);
                    float sigmaVal = (tmpError == 0) ? 1 : (float)rgbSize;
                    int brk = 0;
                    if (tp.rgbOnly && tmpError > st->lastRGBError) brk = 1;
                    else {
                        st->lastRGBError = tmpError; st->lastRGBCount = (float)rgbSize;
                        if (tp.rgbOnly) sigmaVal = -1;
                        st->sigmaVal = sigmaVal;
                    }
                    flag = brk;
                }
                __syncthreads();
                if (flag) break;                                        // uniform over the whole grid: every CTA holds the same state
                // ---- phase B: photometric normal equations with the weights of this iteration ----
                double fR[2] = {0.0, 0.0};
                if (active) {
                    const float sigmaSh = st->sigmaVal;
                    auto rgbRow = [&](int2 c, short2 g, float4 cp, float* row) {
                        const float diff = __int_as_float(c.y);
                        float w = sigmaSh + fabsf(diff);
                        w = w > 1.19209290E-07F ? 1.0f / w : 1.0f;
                        if (sigmaSh == -1) w = 1;
                        const float invz = cp.w;                           // (float)(1.0 / (double)cp.z), precomputed by k_project_points3
                        float dIdx_v = w * tp.sobelScale * (float)g.x;      // grad[one]: `one` is this pixel (reduce.cu:934)
                        float dIdy_v = w * tp.sobelScale * (float)g.y;
                        float v0 = dIdx_v * cam.fx * invz;
                        float v1 = dIdy_v * cam.fy * invz;
                        float v2 = -(v0 * cp.x + v1 * cp.y) * invz;
                        putRow(row, make_float4(v0, v1, v2, -cp.z * v1 + cp.y * v2), make_float4(cp.z * v0 - cp.x * v2, -cp.y * v0 + cp.x * v1, -w * diff, 0.f));
                    };
                    for (int r = 0; r < roundsW; r += 2) {
                        const bool hasA = r < rounds, hasB = r + 1 < rounds;
                        const int k0 = hasA ? kOf(r) : 0, k1 = hasB ? kOf(r + 1) : k0;
                        const int2 c0 = hasA ? corr[r * PT_THREADS + threadIdx.x] : make_int2(-1, 0);
                        const int2 c1 = hasB ? corr[(r + 1) * PT_THREADS + threadIdx.x] : make_int2(-1, 0);
                        short2 g0 = make_short2(0, 0), g1 = g0;
                        float4 p0 = make_float4(0, 0, 1, 0), p1 = p0;
                        auto gradOf = [&](int k, int rr) -> short2 {
                            if (rr < cRounds) { const uint32_t g = gS[rr * PT_THREADS + threadIdx.x]; return make_short2((short)(g & 0xffffu), (short)(g >> 16)); }
                            return grad[k];
                        };
                        if (c0.x != -1) { g0 = gradOf(k0, r); p0 = cloud[(c0.x >> 16) * W + (c0.x & 0xffff)]; }
                        if (c1.x != -1) { g1 = gradOf(k1, r + 1); p1 = cloud[(c1.x >> 16) * W + (c1.x & 0xffff)]; }
                        if (c0.x != -1) rgbRow(c0, g0, p0, tiles[0][threadIdx.x & 31]);
                        if (c1.x != -1) rgbRow(c1, g1, p1, tiles[1][threadIdx.x & 31]);
                        warpAccumulate(tiles[0], c0.x != -1, fR);
                        warpAccumulate(tiles[1], c1.x != -1, fR);
                    }
                }
                TT(6);
                // the next iteration's first pixel pair (pose-independent inputs) -> L1 across the reduction and the solve
                for (int q = cRounds; q < cRounds + 2; ++q)
                    if (q < rounds) {
                        const int kn = kOf(q);
                        if (tp.icp) { prefetchL1(vmapC + kn); prefetchL1(nmapC + kn); }
                        prefetchL1(nextDepth + kn);
                    }
                // ICP totals stay in tot[0..28]; the photometric ones go behind them
                reduceStep<7, NACC_RGB>(fR, 0, 0, active, rc, wsc, ws, totR);
                TT(9);
                if (threadIdx.x < NACC_RGB) tot[NACC_ICP + threadIdx.x] = totR[threadIdx.x];
                __syncthreads();
            }
            if (threadIdx.x < 32) solveAndUpdate(st, tot, tp.icp != 0, tp.rgb != 0, tp.icpWeight, cam, &sc);
            __syncthreads();
            TT(10);
        }
        __syncthreads();
    }

    TT(99);
    // ---------------- result (RGBDOdometry.cpp:478-497) ----------------
    if (bx == 0 && threadIdx.x == 0) {
        float dx = st->tcurr[0] - st->tprev[0], dy = st->tcurr[1] - st->tprev[1], dz = st->tcurr[2] - st->tprev[2];
        if (tp.rgb && sqrtf((dx * dx + dy * dy) + dz * dz) > 0.3f) {          // :478-482
            for (int k = 0; k < 9; ++k) { st->Rcurr[k] = st->Rprev[k]; st->trR[k] = (k % 4 == 0) ? 1.f : 0.f; }
            for (int k = 0; k < 3; ++k) { st->tcurr[k] = st->tprev[k]; st->trT[k] = 0; }
        }
        float* po = st->out;                 // [0..15] pose, [16..31] transform, [32..37] error stats
        for (int k = 0; k < 32; ++k) po[k] = ((k % 16) % 5 == 0) ? 1.f : 0.f;
        for (int r = 0; r < 3; ++r) {
            for (int c = 0; c < 3; ++c) { po[r * 4 + c] = st->Rcurr[r * 3 + c]; po[16 + r * 4 + c] = st->trR[r * 3 + c]; }
            po[r * 4 + 3] = st->tcurr[r]; po[16 + r * 4 + 3] = st->trT[r];
        }
        po[32] = st->lastICPError; po[33] = st->lastICPCount; po[34] = st->lastRGBError; po[35] = st->lastRGBCount;
        po[36] = st->lastSO3Error; po[37] = st->lastSO3Count;
        *J.st = *st;
        // device-resident pose for the passes that follow (index map, association, clean, splat): no host round trip
        float last[16];
        for (int k = 0; k < 16; ++k) last[k] = (k % 5 == 0) ? 1.f : 0.f;
        for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) last[r * 4 + c] = st->Rprev[r * 3 + c]; last[r * 4 + 3] = st->tprev[r]; }
        derivePose(J.dpose, po, last);
    }
}

// ------------------------------ host launchers ----------------------------------------
float track_min_scale(int level)
{
    const float minGrad[3] = {5, 3, 1};
    const float sobelScale = (float)(1.0 / 8.0);
    return (float)(pow((double)minGrad[level], 2.0) / pow((double)sobelScale, 2.0));
}

static int trackBlocks(int N)
{
    int need = (N + TRK_THREADS - 1) / TRK_THREADS;
    int cap = num_sms() * 2;
    if (cap > TRACK_MAX_BLOCKS) cap = TRACK_MAX_BLOCKS;
    return need < cap ? need : cap;
}

// CTAs of the persistent tracking grid per model (host logic, exported as mf_track_shares for the CPU tests).  A light model (bit set in
// lightMask: an object model with a validity bitmask) gets one share, a heavy one (full-frame maps) `ratio` shares (launch_tracking passes 2, the
// fastest of 1, 2, 3 and 5 on the 8- and 3-object scenes).  Without both kinds in the batch, or when the grid is too small for 4 CTAs per light model, the shares are equal.
void track_shares(int nJobs, unsigned lightMask, int totalCTAs, int ratio, int* G)
{
    if (nJobs < 1) return;
    int Geq = totalCTAs / nJobs;
    if (Geq > TRACK_MAX_BLOCKS / 2) Geq = TRACK_MAX_BLOCKS / 2;
    int nLight = 0;
    for (int j = 0; j < nJobs; ++j) nLight += (lightMask >> j) & 1u;
    const int nHeavy = nJobs - nLight;
    int Gheavy = Geq, Glight = Geq;
    if (nLight > 0 && nHeavy > 0) {
        Glight = std::max(4, totalCTAs / (nLight + std::max(1, ratio) * nHeavy));
        Gheavy = (totalCTAs - nLight * Glight) / nHeavy;
        if (Gheavy < Glight) { Gheavy = Geq; Glight = Geq; }
        if (Gheavy > TRACK_MAX_BLOCKS / 2) Gheavy = TRACK_MAX_BLOCKS / 2;
    }
    for (int j = 0; j < nJobs; ++j) G[j] = ((lightMask >> j) & 1u) ? Glight : Gheavy;
}

// launch limits of the persistent tracking kernel on one device: CTAs that fit on it at once, and the dynamic shared memory it is opted in for
struct TrackLimits { int coResident; size_t dynMax; };

void launch_tracking(TrackJob* d_jobs, int nJobs, int W, int H, Cam cam, bool rgbOnly, float icpWeight,
                     bool pyramid, bool fastOdom, bool so3, unsigned epoch, Enq q, unsigned lightMask)
{
    const bool anyValidBits = lightMask != 0;          // bit j: job j is an object model with a validity bitmask (nearly all of its pixels are rejected early)
    static PerDevice<TrackLimits> limits([](int dev) {
        int perSM = 0;
        cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSM, k_track_persistent, PT_THREADS, 0);
        if (e != cudaSuccess || perSM < 1) throw CudaError{std::string("k_track_persistent does not fit on an SM: ") + cudaGetErrorString(e)};
        int optin = 0; cudaCheck(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev), "cudaDeviceGetAttribute");
        cudaFuncAttributes fa; cudaCheck(cudaFuncGetAttributes(&fa, k_track_persistent), "cudaFuncGetAttributes");
        TrackLimits l{perSM * num_sms(), (size_t)optin > fa.sharedSizeBytes + 2048 ? (size_t)optin - fa.sharedSizeBytes - 2048 : 0};
        cudaCheck(cudaFuncSetAttribute(k_track_persistent, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)l.dynMax), "cudaFuncSetAttribute");
        return l;
    });
    const TrackLimits& lim = limits.get();
    const int numSMs = num_sms(), coResident = lim.coResident;
    TrackParams tp;
    tp.W = W; tp.H = H; tp.cam = cam;
    tp.icp = (!rgbOnly && icpWeight > 0) ? 1 : 0;
    tp.rgb = (rgbOnly || icpWeight < 100) ? 1 : 0;
    tp.rgbOnly = rgbOnly ? 1 : 0; tp.so3 = so3 ? 1 : 0;
    tp.iterations[0] = fastOdom ? 3 : 10; tp.iterations[1] = pyramid ? 5 : 0; tp.iterations[2] = pyramid ? 4 : 0;
    tp.icpWeight = icpWeight;
    tp.angleThres = (float)sin(20.f * 3.14159254f / 180.f);
    tp.distThres = 0.10f; tp.sobelScale = (float)(1.0 / 8.0); tp.maxDepthDelta = 0.07f;
    for (int l = 0; l < 3; ++l) tp.minScale[l] = track_min_scale(l);
    tp.llBase = epoch << 6;                      // every launch owns 64 flag values
    int G = numSMs / nJobs;                      // one CTA per SM, the SMs split between the tracked models
    if (G * nJobs > coResident) G = coResident / nJobs;
    if (G > TRACK_MAX_BLOCKS / 2) G = TRACK_MAX_BLOCKS / 2;
    if (G < 1) throw CudaError{"too many tracked models for one cooperative launch"};
    // Per-model shares of the persistent grid.  A full-frame model (the background) pays the whole pixel phase for every live pixel; an
    // object model rejects nearly every pixel on its bitmask and is bound by the reduction / solve chain instead: with equal shares the
    // background of the 8-object scene walked 37 pixels per thread while the objects' CTAs idled at their exchanges.  Light models get a
    // small fixed share, the heavy ones split the rest.  (Sums are fp64 of exact products: the result does not depend on the shares.)
    int Gof[TRACK_MAX_JOBS];
    track_shares(nJobs, lightMask, std::min(numSMs, coResident), 2, Gof);
    int Gheavy = 0;                  // the largest share (sizes the shared-memory correspondences)
    for (int j = 0; j < nJobs; ++j) Gheavy = std::max(Gheavy, Gof[j]);
    tp.nJobs = nJobs; tp.jobStart[0] = 0;
    for (int j = 0; j < nJobs; ++j) tp.jobStart[j + 1] = (unsigned short)(tp.jobStart[j] + Gof[j]);
    const int gridCTAs = tp.jobStart[nJobs];
    // photometric correspondences stay in shared memory when the per-CTA pixel share fits (8 B per pixel slot)
    // sized for the models with the largest share (the heavy ones); a CTA whose share needs more slots uses its model's global scratch stripe
    const int rounds0 = (W * H + Gheavy * PT_THREADS - 1) / (Gheavy * PT_THREADS);
    size_t dyn = (size_t)rounds0 * PT_THREADS * sizeof(int2);
    if (tp.rgb && dyn <= lim.dynMax) tp.corrSlots = rounds0 * PT_THREADS; else { tp.corrSlots = 0; dyn = 0; }
    dyn = (dyn + 15) & ~(size_t)15;
    // shared-memory words for the bitmask of a level: only when a job carries one (object models) and it fits behind the correspondences
    tp.bitWords = anyValidBits ? (W * H + 31) / 32 : 0;
    const size_t bitBytes = ((size_t)tp.bitWords * 4 + 15) & ~(size_t)15;
    if (dyn + bitBytes > lim.dynMax) tp.bitWords = 0;
    // MFB200_TRACK_CACHE=0: every iteration re-reads its pose-independent inputs from global memory (A/B)
    static const bool cacheOn = [] { const char* e = getenv("MFB200_TRACK_CACHE"); return e ? e[0] != '0' : MFB200_DEFAULT_TRACK_CACHE != 0; }();
    tp.cacheRounds = cacheOn ? (int)std::min<size_t>((size_t)rounds0, (lim.dynMax - dyn - (tp.bitWords ? bitBytes : 0)) / ((size_t)PT_THREADS * CACHE_BYTES_PER_SLOT)) : 0;
    dyn += (size_t)tp.cacheRounds * PT_THREADS * CACHE_BYTES_PER_SLOT + (tp.bitWords ? bitBytes : 0);
    q.mark("k_track_persistent");
    const TrackJob* jp = d_jobs;
    void* args[] = {(void*)&jp, (void*)&tp};
    cudaLaunchCooperativeKernel((const void*)k_track_persistent, dim3(gridCTAs), dim3(PT_THREADS), args, dyn, q.s);    // a failure is the runtime's last error
    q.launched((const void*)k_track_persistent);
}

// (tag, clock64) pairs of the last tracking launch (A/B build -DMF_TRACK_TIMING only); returns the number of int64 values written
int debug_track_timing(long long* out, int cap)
{
#ifdef MF_TRACK_TIMING
    int n = 0;
    cudaDeviceSynchronize();
    cudaMemcpyFromSymbol(&n, g_trackTimingN, sizeof n);
    if (n > cap) n = cap;
    if (n > 0) cudaMemcpyFromSymbol(out, g_trackTiming, (size_t)n * sizeof(long long));
    return n;
#else
    (void)out; (void)cap;
    return 0;
#endif
}

void launch_icp_only(const float4* vmapC, const float4* nmapC, const float4* vmapG, const float4* nmapG, int W, int H, Cam cam,
                     const TrackPoses& pp, float* partial, unsigned* ticket, float* out29, Enq q)
{
    const float angleThres = (float)sin(20.f * 3.14159254f / 180.f);
    launch(q, "k_icp_only", k_icp_only, trackBlocks(W * H), TRK_THREADS, 0, vmapC, nmapC, vmapG, nmapG, W, H, cam, pp, 0.10f, angleThres,
           reinterpret_cast<double*>(partial), ticket, out29);
}

}  // namespace mfb
