// mf_common.cuh -- shared device helpers for the sm_90a MaskFusion kernels.
//
// Arithmetic contract: every per-element kernel is compiled with -fmad=false and
// uses only IEEE + - * / sqrt, in the operation order written here, so that its
// fp32 outputs are reproducible bit for bit (the parity tests compare against a
// CPU restatement of the reference's shaders/kernels).  exp() and acos(), whose
// precision GLSL leaves implementation-defined, are the fixed polynomials below.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

#define MF_HD __host__ __device__ __forceinline__
#define MF_D __device__ __forceinline__

namespace mfb {

struct Cam { float fx, fy, cx, cy; };
MF_HD Cam camLevel(Cam c, int level) {              // reference: CameraModel::operator(), types.cuh:94-98
    int div = 1 << level;
    return Cam{c.fx / div, c.fy / div, c.cx / div, c.cy / div};
}

// Row-major 3x4 rigid transform [R|t]
struct Rt { float m[12]; };

MF_D float qnanf() { return __int_as_float(0x7fffffff); }   // cudafuncs.cu:130

MF_D float3 xform(const Rt& T, float3 p) {
    return make_float3(((T.m[0] * p.x + T.m[1] * p.y) + T.m[2] * p.z) + T.m[3],
                       ((T.m[4] * p.x + T.m[5] * p.y) + T.m[6] * p.z) + T.m[7],
                       ((T.m[8] * p.x + T.m[9] * p.y) + T.m[10] * p.z) + T.m[11]);
}
MF_D float3 rotate(const Rt& T, float3 n) {
    return make_float3((T.m[0] * n.x + T.m[1] * n.y) + T.m[2] * n.z,
                       (T.m[4] * n.x + T.m[5] * n.y) + T.m[6] * n.z,
                       (T.m[8] * n.x + T.m[9] * n.y) + T.m[10] * n.z);
}
// Rigid-pose arithmetic on row-major 4x4 float arrays, the one definition for the host classes and the kernels.
// Rule R-INV (DESIGN.md): pose.inverse() of a rigid pose is [R^T | -R^T t] in fp32.
MF_HD void rigidInverse(const float* m, float* inv) {
    const float R[9] = {m[0], m[1], m[2], m[4], m[5], m[6], m[8], m[9], m[10]}, t[3] = {m[3], m[7], m[11]};
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) inv[r * 4 + c] = R[c * 3 + r];
        inv[r * 4 + 3] = -((R[0 * 3 + r] * t[0] + R[1 * 3 + r] * t[1]) + R[2 * 3 + r] * t[2]);
    }
    inv[12] = 0.f; inv[13] = 0.f; inv[14] = 0.f; inv[15] = 1.f;
}
// C = A * B, each entry summed as s += A[r][k] * B[k][c], k = 0..3; C must not alias A or B
MF_HD void mul(const float* A, const float* B, float* C) {
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) {
            float s = 0;
            for (int k = 0; k < 4; ++k) s += A[r * 4 + k] * B[k * 4 + c];
            C[r * 4 + c] = s;
        }
}
// Model::rodrigues2 (Model.cpp:890-932) without the SVD re-orthonormalisation (rule R-SVD, DESIGN.md); R row-major 3x3
MF_HD void rodrigues2(const float* R, float* out) {
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
// Model::computeFusionWeight(1.0) (Model.cpp:449-464): max(1 - min(max(|t|, |rotation vector|), 0.01) / 0.01, 0.5) of the last motion
// pose^-1 * lastPose; poseInv = rigidInverse(pose)
MF_HD float fusionWeight(const float* poseInv, const float* last) {
    float diff[16];
    mul(poseInv, last, diff);
    const float R[9] = {diff[0], diff[1], diff[2], diff[4], diff[5], diff[6], diff[8], diff[9], diff[10]};
    float tn = sqrtf((diff[3] * diff[3] + diff[7] * diff[7]) + diff[11] * diff[11]);
    float rv[3]; rodrigues2(R, rv);
    float rn = sqrtf((rv[0] * rv[0] + rv[1] * rv[1]) + rv[2] * rv[2]);
    float weighting = tn > rn ? tn : rn;
    const float largest = 0.01f, minWeight = 0.5f;
    if (weighting > largest) weighting = largest;
    float w = 1.0f - (weighting / largest);
    return w > minWeight ? w : minWeight;
}

MF_D float dot3(float3 a, float3 b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }
MF_D float3 cross3(float3 a, float3 b) {
    return make_float3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}
MF_D float3 normalize3(float3 v) {
    float l = sqrtf(dot3(v, v));
    return make_float3(v.x / l, v.y / l, v.z / l);
}
MF_D float3 sub3(float3 a, float3 b) { return make_float3(a.x - b.x, a.y - b.y, a.z - b.z); }
MF_D float3 add3(float3 a, float3 b) { return make_float3(a.x + b.x, a.y + b.y, a.z + b.z); }

// exp(x): Cody-Waite reduction + degree-6 polynomial (Cephes expf coefficients)
MF_D float det_expf(float x) {
    // the two range cases are applied as selects AFTER the (always evaluated) polynomial: no branches in the 169-tap loops
    const float xin = x;
    x = fminf(fmaxf(x, -87.0f), 88.0f);                 // keeps n + 127 in range for the discarded evaluations (NaN -> -87)
    float t = x * 1.44269504088896341f;
    float n = floorf(t + 0.5f);
    float r = (x - n * 0.693359375f) - n * (-2.12194440e-4f);
    float p = 1.9875691500e-4f;
    p = p * r + 1.3981999507e-3f;
    p = p * r + 8.3334519073e-3f;
    p = p * r + 4.1665795894e-2f;
    p = p * r + 1.6666665459e-1f;
    p = p * r + 5.0000001201e-1f;
    float r2 = r * r;
    float y = (p * r2 + r) + 1.0f;
    float res = y * __int_as_float((uint32_t)((int)n + 127) << 23);
    if (xin > 88.0f) res = __int_as_float(0x7f800000);
    if (!(xin > -87.0f)) res = (xin != xin) ? xin : 0.0f;
    return res;
}
// acos(x): Abramowitz & Stegun 4.4.46
MF_D float det_acosf(float x) {
    float a = fabsf(x);
    if (!(a <= 1.0f)) return qnanf();
    float p = -0.0012624911f;
    p = p * a + 0.0066700901f;
    p = p * a + -0.0170881256f;
    p = p * a + 0.0308918810f;
    p = p * a + -0.0501743046f;
    p = p * a + 0.0889789874f;
    p = p * a + -0.2145988016f;
    p = p * a + 1.5707963050f;
    float r = sqrtf(1.0f - a) * p;
    return x < 0.0f ? 3.14159265358979f - r : r;
}

// colour packing of the surfel record (reference: color_encoding.glsl:19-34)
MF_D float encodeColor(float r, float g, float b) {
    int rgb = (int)floorf(r * 255.0f + 0.5f);
    rgb = (rgb << 8) + (int)floorf(g * 255.0f + 0.5f);
    rgb = (rgb << 8) + (int)floorf(b * 255.0f + 0.5f);
    return (float)rgb;
}
MF_D float3 decodeColor(float c) {
    int ci = (int)c;
    return make_float3((float)((ci >> 16) & 0xFF) / 255.0f, (float)((ci >> 8) & 0xFF) / 255.0f, (float)(ci & 0xFF) / 255.0f);
}
// surfel radius / confidence (reference: surfels.glsl:19-46)
MF_D float surfelRadius(float depth, float norm_z, float ifx, float ify) {
    float meanFocal = ((1.0f / fabsf(ifx)) + (1.0f / fabsf(ify))) / 2.0f;
    float radius = (depth / meanFocal) * 1.41421356237f;
    float radius_n = radius / fabsf(norm_z);
    float r2 = 2.0f * radius;
    return r2 < radius_n ? r2 : radius_n;
}
MF_D float surfelConfidence(float x, float y, float weighting, float cx, float cy) {
    float px = x - cx, py = y - cy;
    float radialDist = sqrtf(px * px + py * py) / 400.0f;
    return det_expf((-(radialDist * radialDist) / 0.72f)) * weighting;
}

MF_D int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// streaming 128-bit accessors: surfel planes are read once per pass (no L1 reuse)
MF_D float4 ldStream(const float4* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
MF_D void stStream(float4* p, float4 v) {
    asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

constexpr uint64_t KEY_EMPTY = ~0ull;

}  // namespace mfb
