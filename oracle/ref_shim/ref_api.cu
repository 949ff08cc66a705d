// oracle/ref_shim/ref_api.cu -- TEST INFRASTRUCTURE (GPU-side oracle): a flat C wrapper
// around the reference's OWN CUDA entry points (Core/Cuda/cudafuncs.cuh:64-193,
// segmentation.cuh:28-52), compiled from the sources where they lie under /root/reference
// by oracle/Makefile.ref into oracle/_ref/libmf_ref.so.  Host arrays in, host arrays out
// (planar 3*rows x cols maps, exactly the reference's DeviceArray2D contents).  Used by
// tests/test_gpu_ref.py to pin the CPU oracle against the reference's kernels on the GPU.
#include "cudafuncs.cuh"
#include "segmentation.cuh"
#include <cstring>
#include <vector>

static mat33 toMat(const float* R) { mat33 m; for (int r = 0; r < 3; ++r) m.data[r] = make_float3(R[r * 3], R[r * 3 + 1], R[r * 3 + 2]); return m; }

extern "C" {

int ref_vmap_nmap(const float* depth, int W, int H, float fx, float fy, float cx, float cy, float cutoff, float* vmap, float* nmap)
{
    DeviceArray2D<float> d, v, n;
    d.upload(depth, W * sizeof(float), H, W);
    v.create(H * 3, W); n.create(H * 3, W);
    cudaMemset2D(v.ptr(), v.step(), 0, W * sizeof(float), H * 3);      // the kernels leave stale planes untouched
    cudaMemset2D(n.ptr(), n.step(), 0, W * sizeof(float), H * 3);
    createVMap(CameraModel(fx, fy, cx, cy), d, v, cutoff);
    createNMap(v, n);
    cudaDeviceSynchronize();
    v.download(vmap, W * sizeof(float)); n.download(nmap, W * sizeof(float));
    return (int)cudaGetLastError();
}

int ref_pyrdown_f(const float* src, int sw, int sh, float* dst)
{
    DeviceArray2D<float> s, d;
    s.upload(src, sw * sizeof(float), sh, sw);
    pyrDownGaussF(s, d);
    cudaDeviceSynchronize();
    d.download(dst, (sw / 2) * sizeof(float));
    return (int)cudaGetLastError();
}
int ref_pyrdown_u8(const unsigned char* src, int sw, int sh, unsigned char* dst)
{
    DeviceArray2D<unsigned char> s, d;
    s.upload(src, sw, sh, sw);
    pyrDownUcharGauss(s, d);
    cudaDeviceSynchronize();
    d.download(dst, sw / 2);
    return (int)cudaGetLastError();
}

// copyMaps + resize x2 + tranformMaps, i.e. RGBDOdometry::initICPModel (RGBDOdometry.cpp:153-185)
int ref_model_maps(const float* vtex4, const float* ntex4, int W, int H, const float* R9, const float* t3, float** vout, float** nout)
{
    DeviceArray<float> vt, nt;
    vt.upload(vtex4, (size_t)W * H * 4); nt.upload(ntex4, (size_t)W * H * 4);
    DeviceArray2D<float> v[3], n[3];
    for (int l = 0; l < 3; ++l) { v[l].create((H >> l) * 3, W >> l); n[l].create((H >> l) * 3, W >> l); }
    copyMaps(vt, nt, v[0], n[0]);
    for (int l = 1; l < 3; ++l) {
        cudaMemset2D(v[l].ptr(), v[l].step(), 0, (W >> l) * sizeof(float), (H >> l) * 3);
        cudaMemset2D(n[l].ptr(), n[l].step(), 0, (W >> l) * sizeof(float), (H >> l) * 3);
        resizeVMap(v[l - 1], v[l]); resizeNMap(n[l - 1], n[l]);
    }
    mat33 R = toMat(R9); float3 t = make_float3(t3[0], t3[1], t3[2]);
    for (int l = 0; l < 3; ++l) tranformMaps(v[l], n[l], R, t, v[l], n[l]);
    cudaDeviceSynchronize();
    for (int l = 0; l < 3; ++l) { v[l].download(vout[l], (W >> l) * sizeof(float)); n[l].download(nout[l], (W >> l) * sizeof(float)); }
    return (int)cudaGetLastError();
}

int ref_icp_step(const float* Rcurr9, const float* tcurr3, const float* vmap_curr, const float* nmap_curr, const float* Rprev_inv9,
                 const float* tprev3, float fx, float fy, float cx, float cy, const float* vmap_g, const float* nmap_g, float distThres,
                 float angleThres, int W, int H, int threads, int blocks, float* A36, float* b6, float* res2)
{
    DeviceArray2D<float> vc, nc, vg, ng;
    vc.upload(vmap_curr, W * sizeof(float), H * 3, W); nc.upload(nmap_curr, W * sizeof(float), H * 3, W);
    vg.upload(vmap_g, W * sizeof(float), H * 3, W); ng.upload(nmap_g, W * sizeof(float), H * 3, W);
    DeviceArray<JtJJtrSE3> sum, out; sum.create(MAX_THREADS); out.create(1);
    DeviceArray2D<unsigned char> mask; mask.create(H, W);
    icpStep(toMat(Rcurr9), make_float3(tcurr3[0], tcurr3[1], tcurr3[2]), vc, nc, toMat(Rprev_inv9), make_float3(tprev3[0], tprev3[1], tprev3[2]),
            CameraModel(fx, fy, cx, cy), vg, ng, distThres, angleThres, sum, out, A36, b6, res2, threads, blocks, 0, mask, 0);
    return (int)cudaGetLastError();
}

// The reference's own calling pattern for the ICP term (RGBDOdometry.cpp:403-430): one icpStep per Gauss-Newton iteration, each with its
// two launches, cudaDeviceSynchronize and 116-byte D2H inside (reduce.cu:446-525).  `iters` calls on resident maps, timed with CUDA events:
// the "reference's own CUDA kernels on this GPU" baseline for the tracker (SURVEY 8d-iii).  Returns ms per call, < 0 on error.
float ref_icp_step_time_ms(const float* Rcurr9, const float* tcurr3, const float* vmap_curr, const float* nmap_curr, const float* Rprev_inv9,
                           const float* tprev3, float fx, float fy, float cx, float cy, const float* vmap_g, const float* nmap_g, float distThres,
                           float angleThres, int W, int H, int threads, int blocks, int iters)
{
    DeviceArray2D<float> vc, nc, vg, ng;
    vc.upload(vmap_curr, W * sizeof(float), H * 3, W); nc.upload(nmap_curr, W * sizeof(float), H * 3, W);
    vg.upload(vmap_g, W * sizeof(float), H * 3, W); ng.upload(nmap_g, W * sizeof(float), H * 3, W);
    DeviceArray<JtJJtrSE3> sum, out; sum.create(MAX_THREADS); out.create(1);
    DeviceArray2D<unsigned char> mask; mask.create(H, W);
    float A36[36], b6[6], res2[2];
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    for (int w = 0; w < 3; ++w)
        icpStep(toMat(Rcurr9), make_float3(tcurr3[0], tcurr3[1], tcurr3[2]), vc, nc, toMat(Rprev_inv9), make_float3(tprev3[0], tprev3[1], tprev3[2]),
                CameraModel(fx, fy, cx, cy), vg, ng, distThres, angleThres, sum, out, A36, b6, res2, threads, blocks, 0, mask, 0);
    cudaEventRecord(e0);
    for (int i = 0; i < iters; ++i)
        icpStep(toMat(Rcurr9), make_float3(tcurr3[0], tcurr3[1], tcurr3[2]), vc, nc, toMat(Rprev_inv9), make_float3(tprev3[0], tprev3[1], tprev3[2]),
                CameraModel(fx, fy, cx, cy), vg, ng, distThres, angleThres, sum, out, A36, b6, res2, threads, blocks, 0, mask, 0);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    return cudaGetLastError() == cudaSuccess ? ms / (float)iters : -1.f;
}

int ref_sobel(const unsigned char* img, int W, int H, short* dx, short* dy)
{
    DeviceArray2D<unsigned char> s; DeviceArray2D<short> gx, gy;
    s.upload(img, W, H, W); gx.create(H, W); gy.create(H, W);
    computeDerivativeImages(s, gx, gy);
    gx.download(dx, W * sizeof(short)); gy.download(dy, W * sizeof(short));
    return (int)cudaGetLastError();
}

int ref_so3_step(const unsigned char* lastImage, const unsigned char* nextImage, const float* basis9, const float* kinv9, const float* krlr9,
                 int W, int H, int threads, int blocks, float* A9, float* b3, float* res2)
{
    DeviceArray2D<unsigned char> a, b;
    a.upload(lastImage, W, H, W); b.upload(nextImage, W, H, W);
    DeviceArray<JtJJtrSO3> sum, out; sum.create(MAX_THREADS); out.create(1);
    so3Step(a, b, toMat(basis9), toMat(kinv9), toMat(krlr9), sum, out, A9, b3, res2, threads, blocks);
    return (int)cudaGetLastError();
}

// computeRgbResidual + rgbStep for one iteration (RGBDOdometry.cpp:381-437)
int ref_rgb_iteration(float minScale, const short* dIdx, const short* dIdy, const float* lastDepth, const float* nextDepth,
                      const unsigned char* lastImage, const unsigned char* nextImage, float maxDepthDelta, const float* kt3, const float* krk9,
                      float sigmaOverride, float fx, float fy, float cx, float cy, int level, float sobelScale, int W, int H,
                      int* count, int* sigmaSum, float* A36, float* b6)
{
    DeviceArray2D<short> gx, gy; gx.upload(dIdx, W * sizeof(short), H, W); gy.upload(dIdy, W * sizeof(short), H, W);
    DeviceArray2D<float> ld, nd; ld.upload(lastDepth, W * sizeof(float), H, W); nd.upload(nextDepth, W * sizeof(float), H, W);
    DeviceArray2D<unsigned char> li, ni, m; li.upload(lastImage, W, H, W); ni.upload(nextImage, W, H, W); m.create(H, W);
    DeviceArray2D<DataTerm> corres; corres.create(H, W);
    DeviceArray<int2> sumRes; sumRes.create(MAX_THREADS);
    computeRgbResidual(minScale, gx, gy, ld, nd, li, ni, m, m, corres, sumRes, maxDepthDelta, make_float3(kt3[0], kt3[1], kt3[2]), toMat(krk9),
                       *sigmaSum, *count, 256, 336, 0, 0);
    DeviceArray2D<float3> cloud; cloud.create(H, W);
    CameraModel intr(fx * (1 << level), fy * (1 << level), cx * (1 << level), cy * (1 << level));
    projectToPointCloud(ld, cloud, intr, level);
    DeviceArray<JtJJtrSE3> sum, out; sum.create(MAX_THREADS); out.create(1);
    float sigma = sigmaOverride != 0 ? sigmaOverride : (float)*count;
    rgbStep(corres, sigma, cloud, fx, fy, gx, gy, sobelScale, sum, out, A36, b6, 128, 112);
    return (int)cudaGetLastError();
}

int ref_geometric_edges(const float* vmap, const float* nmap, int W, int H, float wD, float wC, float thr, float* edge, unsigned char* inverted)
{
    DeviceArray2D<float> v, n, e; DeviceArray2D<unsigned char> bin, inv;
    v.upload(vmap, W * sizeof(float), H * 3, W); n.upload(nmap, W * sizeof(float), H * 3, W);
    e.create(H, W); bin.create(H, W); inv.create(H, W);
    computeGeometricSegmentationMap(v, n, e, wD, wC);
    thresholdMap(e, bin, thr);
    invertMap(bin, inv);
    cudaDeviceSynchronize();
    e.download(edge, W * sizeof(float)); inv.download(inverted, W);
    return (int)cudaGetLastError();
}


// SURVEY 8(d)(iii) "B-ref-cuda": the reference's OWN kernels for one model-frame of tracking, in the reference's calling pattern
// (RGBDOdometry.cpp:153-225, 254-476; GPUConfig.h:51-58 fallback launch shapes): model-map preparation (copyMaps, 2 resizes per map,
// 3 tranformMaps), the photometric pyramids (verticesToDepth, 2+2 pyrDowns, 3 Sobel pairs, 3 projectToPointCloud), <= 10 so3Step on
// level 2, then 4/5/10 iterations of computeRgbResidual + icpStep + rgbStep on levels 2/1/0 -- every call with the launches,
// cudaDeviceSynchronize, cudaMalloc/cudaFree and D2H copies it contains.  The host Eigen solve between the iterations is NOT included
// (a few microseconds; it cannot be compiled here), the pose is held fixed.  Inputs are uploaded once; `reps` repetitions are timed.
// Returns the total milliseconds per model-frame in ms[0] and the parts in ms[1..4] = maps, pyramids, so3, levels.  < 0 on error.
int ref_track_schedule_time_ms(const float* vtex4, const float* ntex4, const float* vmapC[3], const float* nmapC[3], const unsigned char* lastImage0,
                               const unsigned char* nextImage0, const float* R9, const float* t3, float fx, float fy, float cx, float cy, int W, int H,
                               int so3Iters, int reps, float* ms)
{
    DeviceArray<float> vt, nt; vt.upload(vtex4, (size_t)W * H * 4); nt.upload(ntex4, (size_t)W * H * 4);
    DeviceArray2D<float> vg[3], ng[3], vc[3], nc[3], lastDepth[3], nextDepth[3];
    DeviceArray2D<unsigned char> lastImg[3], nextImg[3], mask[3];
    DeviceArray2D<short> gx[3], gy[3];
    DeviceArray2D<float3> cloud[3];
    DeviceArray2D<DataTerm> corres[3];
    for (int l = 0; l < 3; ++l) {
        const int w = W >> l, h = H >> l;
        vg[l].create(h * 3, w); ng[l].create(h * 3, w);
        vc[l].upload(vmapC[l], w * sizeof(float), h * 3, w); nc[l].upload(nmapC[l], w * sizeof(float), h * 3, w);
        lastDepth[l].create(h, w); nextDepth[l].create(h, w); lastImg[l].create(h, w); nextImg[l].create(h, w); mask[l].create(h, w);
        gx[l].create(h, w); gy[l].create(h, w); cloud[l].create(h, w); corres[l].create(h, w);
    }
    lastImg[0].upload(lastImage0, W, H, W); nextImg[0].upload(nextImage0, W, H, W);
    DeviceArray<JtJJtrSE3> sumSE3, outSE3; sumSE3.create(MAX_THREADS); outSE3.create(1);
    DeviceArray<JtJJtrSO3> sumSO3, outSO3; sumSO3.create(MAX_THREADS); outSO3.create(1);
    DeviceArray<int2> sumRes; sumRes.create(MAX_THREADS);
    const mat33 R = toMat(R9); const float3 t = make_float3(t3[0], t3[1], t3[2]);
    float Ri9[9]; for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) Ri9[r * 3 + c] = R9[c * 3 + r];
    const mat33 Rinv = toMat(Ri9);
    const float I9[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    float A36[36], b6[6], res2[2], A9[9], b3[3];
    const int iterations[3] = {10, 5, 4};
    const float minGrad[3] = {5, 3, 1};
    const float sobelScale = 1.0f / 8.0f;
    cudaEvent_t e[5]; for (int k = 0; k < 5; ++k) cudaEventCreate(&e[k]);
    float acc[5] = {0, 0, 0, 0, 0};
    for (int rep = -1; rep < reps; ++rep) {                        // rep -1: warm-up
        cudaEventRecord(e[0]);
        // RGBDOdometry::initICPModel (RGBDOdometry.cpp:153-185)
        copyMaps(vt, nt, vg[0], ng[0]);
        for (int l = 1; l < 3; ++l) { resizeVMap(vg[l - 1], vg[l]); resizeNMap(ng[l - 1], ng[l]); }
        for (int l = 0; l < 3; ++l) tranformMaps(vg[l], ng[l], R, t, vg[l], ng[l]);
        cudaDeviceSynchronize();
        cudaEventRecord(e[1]);
        // populateRGBDData x2 + derivative images + clouds (RGBDOdometry.cpp:187-225, 245-250, 349); the BGR->intensity kernel reads a
        // texture reference that CUDA 12 removed, so the intensity images are given
        verticesToDepth(vt, lastDepth[0], 6.0f); verticesToDepth(vt, nextDepth[0], 6.0f);
        for (int l = 0; l + 1 < 3; ++l) {
            pyrDownGaussF(lastDepth[l], lastDepth[l + 1]); pyrDownGaussF(nextDepth[l], nextDepth[l + 1]);
            pyrDownUcharGauss(lastImg[l], lastImg[l + 1]); pyrDownUcharGauss(nextImg[l], nextImg[l + 1]);
        }
        for (int l = 0; l < 3; ++l) computeDerivativeImages(nextImg[l], gx[l], gy[l]);
        for (int l = 0; l < 3; ++l) { CameraModel intr(fx, fy, cx, cy); projectToPointCloud(lastDepth[l], cloud[l], intr, l); }
        cudaDeviceSynchronize();
        cudaEventRecord(e[2]);
        // SO(3) pre-alignment (RGBDOdometry.cpp:272-345), level 2
        {
            const int l = 2; const float s = 1.0f / (1 << l);
            const float K[9] = {fx * s, 0, cx * s, 0, fy * s, cy * s, 0, 0, 1};
            const float Kinv[9] = {1 / (fx * s), 0, -cx / fx, 0, 1 / (fy * s), -cy / fy, 0, 0, 1};
            for (int i = 0; i < so3Iters; ++i) so3Step(lastImg[l], nextImg[l], toMat(I9), toMat(Kinv), toMat(K), sumSO3, outSO3, A9, b3, res2, 160, 64);
        }
        cudaEventRecord(e[3]);
        // pyramid levels (RGBDOdometry.cpp:347-476)
        for (int l = 2; l >= 0; --l) {
            const float s = 1.0f / (1 << l);
            const CameraModel intr(fx * s, fy * s, cx * s, cy * s);
            const float kt[3] = {0, 0, 0};
            const float minScale = (minGrad[l] * minGrad[l]) / (sobelScale * sobelScale);
            for (int j = 0; j < iterations[l]; ++j) {
                int sigma = 0, count = 0;
                computeRgbResidual(minScale, gx[l], gy[l], lastDepth[l], nextDepth[l], lastImg[l], nextImg[l], mask[l], mask[l], corres[l], sumRes, 0.07f,
                                   make_float3(kt[0], kt[1], kt[2]), toMat(I9), sigma, count, 256, 336, 0, 0);
                icpStep(R, t, vc[l], nc[l], Rinv, t, intr, vg[l], ng[l], 0.10f, 0.342020143f, sumSE3, outSE3, A36, b6, res2, 128, 112, 0, mask[l], 0);
                rgbStep(corres[l], (float)(count > 0 ? count : 1), cloud[l], intr.fx, intr.fy, gx[l], gy[l], sobelScale, sumSE3, outSE3, A36, b6, 128, 112);
            }
        }
        cudaDeviceSynchronize();
        cudaEventRecord(e[4]); cudaEventSynchronize(e[4]);
        if (rep >= 0) for (int k = 0; k < 4; ++k) { float m = 0; cudaEventElapsedTime(&m, e[k], e[k + 1]); acc[k + 1] += m; acc[0] += m; }
    }
    for (int k = 0; k < 5; ++k) { ms[k] = acc[k] / (float)reps; cudaEventDestroy(e[k]); }
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

}  // extern "C"
