// mf_host.cu -- host orchestration of the dense pipeline: MaskFusion::processFrame schedule
// (Core/MaskFusion.cpp:200-607) and the Model methods it drives (Core/Model/Model.cpp).
// Everything is enqueued on one CUDA stream; the only host<->device synchronisation inside
// a frame is the read-back of the tracked poses (one per frame, not one per Gauss-Newton
// iteration as in the reference).
#include "mf_host.h"
#include <math.h>
#include <float.h>
#include <string.h>
#include <stdio.h>
#include <limits.h>
#include <stdlib.h>

namespace mfb {

void cudaCheck(cudaError_t e, const char* where)
{
    if (e != cudaSuccess) throw CudaError{std::string(where) + ": " + cudaGetErrorString(e)};
}

void Enq::mark(const char* name) const
{
    if (!rec || !rec->prof.on) return;
    Profiler* p = &rec->prof;
    if (p->used == (int)p->events.size()) {
        Event e; e.create(cudaEventDefault); p->events.push_back(std::move(e)); p->names.push_back(nullptr);
    }
    p->names[p->used] = name;
    cudaEventRecord(p->events[p->used], s);
    p->used++;
}
void Enq::launched(const void* kernel) const
{
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        const char* fn = nullptr;
        if (cudaFuncGetName(&fn, kernel) != cudaSuccess || !fn) fn = "a kernel";
        throw CudaError{std::string("launch of ") + fn + ": " + cudaGetErrorString(e)};
    }
    if (rec) rec->launches++;
}
void Profiler::resolve()
{
    // caller has synchronised the stream
    for (int i = 0; i + 1 < used; ++i) {
        if (!names[i]) continue;
        float ms = 0;
        if (cudaEventElapsedTime(&ms, events[i], events[i + 1]) == cudaSuccess) { auto& a = acc[names[i]]; a.first += 1; a.second += ms; }
    }
    used = 0;
}

Rt toRt(const Mat4& T) { Rt r; for (int i = 0; i < 12; ++i) r.m[i] = T.m[i]; return r; }

// Eigen::Quaternionf(Matrix3f) as used by the pose log (MaskFusion.cpp:585-590)
static void rotToQuat(const float* R, float* q)
{
    float t = R[0] + R[4] + R[8];
    if (t > 0) {
        t = sqrtf(t + 1.0f); q[3] = 0.5f * t; t = 0.5f / t;
        q[0] = (R[7] - R[5]) * t; q[1] = (R[2] - R[6]) * t; q[2] = (R[3] - R[1]) * t;
    } else {
        int i = 0; if (R[4] > R[0]) i = 1; if (R[8] > R[i * 4]) i = 2;
        int j = (i + 1) % 3, k = (j + 1) % 3;
        t = sqrtf(R[i * 4] - R[j * 4] - R[k * 4] + 1.0f);
        q[i] = 0.5f * t; t = 0.5f / t;
        q[3] = (R[k * 3 + j] - R[j * 3 + k]) * t;
        q[j] = (R[j * 3 + i] + R[i * 3 + j]) * t;
        q[k] = (R[k * 3 + i] + R[i * 3 + k]) * t;
    }
}

// ======================================================================================
// Model
// ======================================================================================
Model::Model(MaskFusion* o, unsigned char id_, float conf, bool enableFillIn, int cap, int ownerRank_, bool ghost)
    : owner(o), ownerRank(ownerRank_), owned(!ghost), id(id_), pose(Mat4::identity()), lastPose(Mat4::identity()), initialC2Winv(Mat4::identity()),
      confidenceThreshold(conf), maxDepth(FLT_MAX), fillIn(enableFillIn), capacity((uint32_t)cap), lastTransform(Mat4::identity())
{
    const int W = o->W, H = o->H, P = o->P;
    cudaStream_t s = o->stream;
    if (ghost) return;
    // in-place clean: ONE copy of the store; Model::clean allocates the second plane set when it first needs the copy
    pos[0].alloc(capacity); col[0].alloc(capacity); nrm[0].alloc(capacity);
    count.alloc(2); count.zero(s);
    hCount.alloc(2);
    hTrackOut.alloc(40);
    key.alloc(P); launch_fill_u64(key, KEY_EMPTY, P, o->on());
    idx.alloc(P); vertConf.alloc(P); colorTime.alloc(P); normRad.alloc(P); cleanTex.alloc((size_t)P); cleanTex.zero(s);
    idx.zero(s); vertConf.zero(s); colorTime.zero(s); normRad.zero(s);
    splatImage.alloc(P); splatVertex.alloc(P); splatNormal.alloc(P); splatTime.alloc(P);
    splatImage.zero(s); splatVertex.zero(s); splatNormal.zero(s); splatTime.zero(s);
    nonBlack.alloc(1); nonBlack.zero(s);
    if (fillIn) { fillImage.alloc(P); fillVertex.alloc(P); fillNormal.alloc(P); fillImage.zero(s); fillVertex.zero(s); fillNormal.zero(s); }
    aflag.alloc(P); abest.alloc(P); aflag.zero(s); abest.zero(s);
    for (int k = 0; k < 3; ++k) { meas[k].alloc(P); meas[k].zero(s); }
    slot.alloc(capacity); launch_fill_u32(slot, 0xffffffffu, capacity, o->on());
    keep.alloc((size_t)capacity + P);
    size_t nblk = ((size_t)capacity + P + 511) / 512 + 1;
    blockSums.alloc(nblk); blockSums2.alloc(nblk);
    cleanTicket.alloc(4); cleanTicket.zero(s); cleanLoaded.alloc(nblk); cleanLoaded.zero(s);
    hCleanStat.alloc(2);
    cand.alloc((size_t)capacity + P); candCount.alloc(1); candCount.zero(s);
    for (int l = 0; l < 3; ++l) {
        size_t Pl = (size_t)(W >> l) * (H >> l);
        vmapG[l].alloc(Pl); nmapG[l].alloc(Pl); cloud[l].alloc(Pl); lastDepth[l].alloc(Pl); lastImage[l].alloc(Pl); corres[l].alloc(l == 0 ? Pl + (size_t)num_sms() * 512 : 1);   // level 0 only: scratch when the correspondences do not fit in shared memory
        vmapG[l].zero(s); nmapG[l].zero(s); lastDepth[l].zero(s); lastImage[l].zero(s);
    }
    if (id_ != 0) for (int l = 0; l < 3; ++l) { validBits[l].alloc(((size_t)(W >> l) * (H >> l) + 31) / 32 + 1); validBits[l].zero(s); }
    lastNextImage2.alloc((size_t)(W >> 2) * (H >> 2)); lastNextImage2.zero(s);
    trackState.alloc(1); trackState.zero(s);
    partial.alloc((size_t)TRACK_MAX_BLOCKS * 128); partial.zero(s);     // 2 x 512 rows x 32 x 16 B (flagged words); flags start at 0: never a valid flag
    dpose.alloc(1); pushPose();
}

void Model::pushPose()
{
    if (!owned || !dpose.p) return;          // ghosts hold no device state; during construction the buffer appears last
    launch_set_pose(dpose, pose.m, lastPose.m, owner->on());
}

unsigned Model::lastCount()
{
    if (!owned) throw CudaError{"model is owned by another rank (sharded mode): no surfel store here"};
    cudaCheck(cudaMemcpyAsync(hCount, dCount(), sizeof(uint32_t), cudaMemcpyDeviceToHost, owner->stream), "count D2H");
    owner->sync();
    return hCount[0];
}

// Model::initialise (Model.cpp:240-285) fed by MaskFusion::computeFeedbackBuffers (MaskFusion.cpp:187-198)
void Model::initialise(int time)
{
    MaskFusion* o = owner;
    launch_init_model(o->rgb, o->depthRaw, o->depthFilt, o->cam, o->W, o->H, time, o->cfg.maxDepthProcessed, o->initFlagR, o->initFlagF,
                      blockSums, blockSums2, capacity, current(), dCount(), o->on());
}

// model side of Model::initICP (Model.cpp:391-409): predicted (or fill-in) maps -> pyramids in the model-global frame
void Model::prepareTracking()
{
    MaskFusion* o = owner;
    const Enq q = o->on();
    const int W = o->W, H = o->H;
    float denom = (float)((H / 20) * (W / 20));
    float4* v[3] = {vmapG[0].p, vmapG[1].p, vmapG[2].p};
    float4* n[3] = {nmapG[0].p, nmapG[1].p, nmapG[2].p};
    const uint32_t* nb = fillIn ? nonBlack.p : nullptr;
    launch_model_maps(splatVertex, splatNormal, fillIn ? fillVertex.p : splatVertex.p, fillIn ? fillNormal.p : splatNormal.p, nb, denom, W, H,
                      dpose, 6.0f /* maxDepthRGB, RGBDOdometry.cpp:34 */, v, n, lastDepth[0], q);
    if (validBits[0].p) {
        uint32_t* b3[3] = {validBits[0].p, validBits[1].p, validBits[2].p};
        launch_valid_bits3(n, W, H, b3, q);
    }
    const bool rgb = o->cfg.rgbOnly || o->cfg.icpWeight < 100;
    if (rgb) {
        launch_intensity_select(splatImage, fillIn ? fillImage.p : splatImage.p, nb, denom, (o->cfg.frameToFrameRGB && fillIn) ? 1 : 0, o->P, lastImage[0], q);
        launch_pyrdown2_pair(lastDepth[0], lastDepth[1], lastDepth[2], lastImage[0], lastImage[1], lastImage[2], W, H, q);
        const float* d3[3] = {lastDepth[0].p, lastDepth[1].p, lastDepth[2].p};
        float4* c3[3] = {cloud[0].p, cloud[1].p, cloud[2].p};
        launch_project_points3(d3, W, H, o->cam, c3, q);
    }
}

void Model::predictIndices(int time, float depthCutoff, int timeDelta, bool forClean)
{
    MaskFusion* o = owner;
    if (forClean) {                                                   // lazily: see idxDeferred
        idxDeferred = true; idxTime = time; idxDelta = timeDelta; idxDepth = depthCutoff;
        return;
    }
    idxDeferred = false;
    launch_predict_indices(current(), dCount(), dpose, o->cam, o->W, o->H, depthCutoff, time, timeDelta, key, idx, vertConf,
                           colorTime, normRad, forClean ? cleanTex.p : nullptr, confidenceThreshold, o->on());
    if (forClean) { cleanTexTime = time; cleanTexConf = confidenceThreshold; }
}

void Model::flushIndex()
{
    if (!idxDeferred) return;
    idxDeferred = false;
    MaskFusion* o = owner;
    launch_predict_indices(current(), dCount(), dpose, o->cam, o->W, o->H, idxDepth, idxTime, idxDelta, key, idx, vertConf, colorTime, normRad, cleanTex.p, confidenceThreshold, o->on());
    cleanTexTime = idxTime; cleanTexConf = confidenceThreshold;
}

void Model::fuse(int time, float depthCutoff, float weightMultiplier)
{
    MaskFusion* o = owner;
    flushIndex();
    float md = depthCutoff < maxDepth ? depthCutoff : maxDepth;      // Model.cpp:527 (headless: bounding box empty, N7)
    float4* m[3] = {meas[0].p, meas[1].p, meas[2].p};
    launch_associate(o->rgb, o->depthRaw, o->depthFilt, o->mask, idx, vertConf, normRad, dpose, o->cam, o->W, o->H, md, time,
                     weightMultiplier, id, aflag, abest, m, slot, o->on());
    launch_fuse_update(aflag, abest, m, slot, o->P, time, current(), o->on());
}

void Model::clean(int time, int timeDelta, float /*depthCutoff*/)
{
    MaskFusion* o = owner;
    float4* m[3] = {meas[0].p, meas[1].p, meas[2].p};
    // In-place compaction moves only the surfels behind the first removal, cheap when removals sit in the young tail of the store (the
    // steady state), but its ticketed hand-over is slower than the copy when most of a large store moves (a removal near the front:
    // e.g. the first frames after a map upload).  Both produce the same store, so the choice is free: a large store uses the copy into
    // a second plane set (allocated on first need) for the frame that FOLLOWS one in which more than 40 % of it moved -- the statistic
    // comes back with an asynchronous 8-byte copy and is read without waiting (a stale value only delays the switch).
    bool pingPong = false;
    if (capacity >= (1u << 20) && hCleanStat[1] > 0) {
        const uint32_t first = hCleanStat[0], nb = hCleanStat[1];
        pingPong = first < nb && (uint64_t)(nb - first) * 10 > (uint64_t)nb * 4;
    }
    if (pingPong && !pos[1 - target].p) { pos[1 - target].alloc(capacity); col[1 - target].alloc(capacity); nrm[1 - target].alloc(capacity); }
    int other = pingPong ? 1 - target : target, otherCount = 1 - countSel;
    // the pending index projection rides in pass 1 when it uses this call's time gate (always, in the frame schedule)
    const bool fused = idxDeferred && idxTime == time && idxDelta == timeDelta && (size_t)capacity + (size_t)o->P < 0x80000000ull;   // bit 31 of a candidate entry is a flag
    if (!fused) flushIndex();
    IndexFused f{key.p, idx.p, vertConf.p, colorTime.p, normRad.p, cleanTex.p, idxDepth};
    idxDeferred = false;
    // the packed window texels carry two tests evaluated with a time and a confidence threshold: valid for this call when the index
    // map is resolved inside it, or was resolved with the same two values (the frame schedule); else the window reads the images
    const bool packedOK = fused || (cleanTexTime == time && cleanTexConf == confidenceThreshold);
    CleanWindowImages win{packedOK ? cleanTex.p : nullptr, vertConf.p, colorTime.p, idx.p};
    if (++cleanEpoch == 0) ++cleanEpoch;                              // 0 = "never published"
    CleanInPlace ip{cleanTicket.p, cleanLoaded.p, cleanTicket.p + 1, cleanEpoch, pingPong};
    launch_clean(planes(target), planes(other), dCount(), count.p + otherCount, capacity, aflag, m, dpose, o->cam, o->W, o->H,
                 time, timeDelta, confidenceThreshold, o->cfg.outlierCoeff, id, win, o->depthFilt, o->mask, keep, blockSums,
                 cand, candCount, o->on(), ip, fused ? &f : nullptr);
    if (capacity >= (1u << 20))
        cudaCheck(cudaMemcpyAsync(hCleanStat, cleanTicket.p + 1, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, o->stream), "clean statistic D2H");
    target = other; countSel = otherCount;
}

void Model::combinedPredict(float depthCutoff, int time, int maxTime, int timeDelta)
{
    MaskFusion* o = owner;
    launch_combined_predict(current(), dCount(), dpose, o->cam, o->W, o->H, depthCutoff, confidenceThreshold, time, maxTime,
                            timeDelta, o->rayTab, key, splatImage, splatVertex, splatNormal, splatTime, fillIn ? 1 : 0, o->depthFilt, o->rgb, 0,
                            o->cfg.frameToFrameRGB ? 1 : 0, fillImage, fillVertex, fillNormal, fillIn ? nonBlack.p : nullptr, o->on(), capacity);
}

// ======================================================================================
// MaskFusion
// ======================================================================================
MaskFusion::MaskFusion(const mf_config& c, int dev, cudaStream_t st) : cfg(c), device(dev)
{
    cudaCheck(cudaSetDevice(dev), "cudaSetDevice");
    W = c.width; H = c.height; P = W * H;
    if (W % 4 || H % 4) throw CudaError{"width and height must be multiples of 4 (3-level pyramid)"};
    cam = Cam{c.fx, c.fy, c.cx, c.cy};
    if (st) stream = st;
    else { ownedStream.create(); stream = ownedStream; }
    for (int k = 0; k < 2; ++k) { ring.emplace_back(new FrameSlot(packetBytes(), stream)); rgbBuf[k].alloc(P); depthFiltBuf[k].alloc(P); }
    selectSlot(0); selectSet(0);
    retired.create();
    mask.alloc(P); mask.zero(stream);
    preStream.create();
    preDone.create(); inputsCopied.create(); evMain.create(); evComm.create(); trackDone.create();
    for (int l = 0; l < 3; ++l) {
        size_t Pl = (size_t)(W >> l) * (H >> l);
        if (l > 0) depthPyr[l].alloc(Pl);
        vmap[l].alloc(Pl); nmap[l].alloc(Pl); nextImage[l].alloc(Pl); nextGrad[l].alloc(Pl); rgbValid[l].alloc(Pl);
    }
    edgeMap.alloc(P); edgeBinary.alloc(P); edgeBuf.alloc(P); edgeInv.alloc(P);
    dJobs.alloc(TRACK_MAX_JOBS);
    hJobs.alloc(TRACK_MAX_JOBS);
    initFlagR.alloc(P); initFlagF.alloc(P);
    scratch.alloc((size_t)P * 4);
    rayTab.alloc(P); launch_ray_table(cam, W, H, rayTab, on());
    if (c.enableMultipleModels) {
        dRes.alloc(1); dRes.zero(stream);
        hRes.alloc(1);
        resEvt.create();
        poseTable.alloc((size_t)MF_MAX_MODELS * 32); poseTable.zero(stream);
        gathered.alloc((size_t)64 * MF_MAX_MODELS * 32); gathered.zero(stream);
        // component histograms for the worst case (every second pixel its own component): the counts of a frame live on the device
        compModel.alloc(((size_t)P / 2 + 2) * MF_MAX_MODELS); compMask.alloc(((size_t)P / 2 + 2) * 256);
        projKeys.alloc(P); launch_fill_u64(projKeys, KEY_EMPTY, P, on()); projectedIDs.alloc(P); projectedIDs.zero(stream);
        ccL.alloc(P); ccDense.alloc(P); ccLabA.alloc(P); ccLabB.alloc(P); ccArea.alloc((size_t)P + 1); ccBox.alloc(((size_t)P / 2 + 2) * 4); mapToMask.alloc((size_t)P / 2 + 2); absorbId.alloc((size_t)P / 2 + 2);
        maskPixels.alloc(256); ccCounter.alloc(1); ccCounter.zero(stream);
        segTmp.alloc(P); ignoreMap.alloc(P); ignoreMap.zero(stream);
        tblIdToIndex.alloc(256); tblIndexToId.alloc(256); tblIsModel.alloc(256); tblMaskToID.alloc(256); tblIsPerson.alloc(256);
        tblIdToIndex.zero(stream); tblIndexToId.zero(stream); tblIsModel.zero(stream); tblIsPerson.zero(stream);
        tblMaskToID.zero(stream); cudaCheck(cudaMemsetAsync(tblMaskToID.p + 255, 255, 1, stream), "memset");   // maskToID[255] = 255, MfSegmentation.cpp:70-71 (persists across frames)
        maskOverlap.alloc((size_t)MF_MAX_MODELS * 256);
    }
    models.emplace_back(new Model(this, nextID++, c.confGlobal, true, c.capacityGlobal));    // MaskFusion.cpp:80-81
    sync();
}

MaskFusion::~MaskFusion()
{
    for (auto& f : ring) if (f->netUsed) cudaEventSynchronize(f->netDone);    // a network still reading a slot or writing its hand-off into one
    cudaStreamSynchronize(stream);
    cudaStreamSynchronize(preStream);
    // the members' owners then release every stream, event and buffer the context holds
}

MaskFusion::FrameSlot::FrameSlot(size_t bytes, cudaStream_t s)
{
    uploaded.create(); netDone.create();
    packet.alloc(bytes); packet.zero(s);
}

// MaskFusion::frameQueue with queueLength (-frameQ, MaskFusion.cpp:37,206-209): before the first frame, in one process
void MaskFusion::setFrameQueue(int length)
{
    if (length < 0) throw CudaError{"setFrameQueue: the queue length must be >= 0 (0 or 1: no queue), got " + std::to_string(length)};
    if (world > 1 || shardNccl) throw CudaError{"setFrameQueue: this context is one rank of an object-sharded run, which runs without a frame queue"};
    if (tick != 1 || queued) throw CudaError{"setFrameQueue: must be called before the first frame"};
    const size_t n = (size_t)(length > 1 ? length : 1) + 1;
    if (n != ring.size()) {
        // the new slots first: on failure the ring stays as it was.  The current slot (what mf_set_frame wrote) is kept as slot 0.
        std::vector<std::unique_ptr<FrameSlot>> fresh;
        try {
            for (size_t k = 1; k < n; ++k) fresh.emplace_back(new FrameSlot(packetBytes(), stream));
        } catch (const CudaError& e) {
            cudaGetLastError();
            throw CudaError{"setFrameQueue: cannot allocate " + std::to_string(n) + " frame slots of " + std::to_string(packetBytes()) + " bytes (" + e.what + ")"};
        }
        waitNetwork();
        fresh.insert(fresh.begin(), std::move(ring[curSlot]));
        ring.swap(fresh);
        selectSlot(0);
    }
    queueLength = length;
}

void MaskFusion::sync()
{
    on().mark(nullptr);                                 // closes the last open interval
    cudaCheck(cudaStreamSynchronize(stream), "cudaStreamSynchronize");
    if (rec.prof.on) rec.prof.resolve();
    finalisePending();
}

// textureRGB / textureDepthMetric (+ FrameData::mask, classIDs) upload into the frame packet of `slot` (MaskFusion.cpp:212-217)
void MaskFusion::uploadInputs(int slot, const uint8_t* rgbIn, const float* depthIn, const uint8_t* maskIn, int64_t timestamp, bool onDevice, cudaStream_t s)
{
    if (!s) s = stream;
    cudaMemcpyKind kind = onDevice ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    on(s).mark(onDevice ? "copy_d2d_frame" : "copy_h2d_frame");
    if (onDevice && inputReady) { cudaCheck(cudaStreamWaitEvent(s, inputReady, 0), "cudaStreamWaitEvent"); inputReady = nullptr; }   // caller's producer
    uint8_t* pk = ring[slot]->packet.p;
    cudaCheck(cudaMemcpyAsync(pk, rgbIn, (size_t)P * 3, kind, s), "rgb upload");
    cudaCheck(cudaMemcpyAsync(pk + (size_t)P * 3, depthIn, (size_t)P * sizeof(float), kind, s), "depth upload");
    if (cfg.enableMultipleModels) {
        // instance masks + their class list ride with the images: the header is a kernel argument (no staging buffer to keep alive)
        FrameHdr h; memset(&h, 0, sizeof h);
        h.timestamp = timestamp;
        h.maskGiven = maskIn != nullptr;
        if (maskIn && !classIDs.empty()) {
            if (classIDs.size() > 256) throw CudaError{"more than 256 mask labels"};
            cudaCheck(cudaMemcpyAsync(slotMask(slot), maskIn, (size_t)P, kind, s), "mask upload");
            h.nMasks = (int)classIDs.size();
            for (size_t i = 0; i < classIDs.size(); ++i) h.classIDs[i] = classIDs[i];
        }
        launch_frame_header(h, slotHdr(slot), on(s));
    }
    // host inputs belong to the caller again when processFrame returns (the reference uploads synchronously): see processFrame.
    // Device inputs copied on the pre-processing stream: the context stream waits for the copies, so whatever the caller queues
    // there after this call (e.g. the producer of the next frame writing the same buffers) is ordered behind them.
    if (!onDevice) { cudaCheck(cudaEventRecord(inputsCopied, s), "cudaEventRecord"); copyPending = true; }
    else if (s != stream) { cudaCheck(cudaEventRecord(inputsCopied, s), "cudaEventRecord"); cudaCheck(cudaStreamWaitEvent(stream, inputsCopied, 0), "cudaStreamWaitEvent"); }
}

// filterDepth (MaskFusion.cpp:650-657) + the RGBA copy every later pass reads
void MaskFusion::preprocess(cudaStream_t s)
{
    launch_unpack_rgb(rgb3, rgb, P, on(s));
    launch_bilateral(depthRaw, depthFilt, W, H, on(s));
    frameMapsValid = false; intensityValid = false;
}

void MaskFusion::setFrame(const uint8_t* rgbIn, const float* depthIn, const uint8_t* maskIn, bool onDevice, cudaStream_t s)
{
    if (!s) s = stream;
    // stage-wise test entry (mf_set_frame): the optional mask goes straight into textureMask like the reference's upload
    if (maskIn) cudaCheck(cudaMemcpyAsync(mask, maskIn, (size_t)P, onDevice ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, s), "mask upload");
    uploadInputs(curSlot, rgbIn, depthIn, nullptr, 0, onDevice, s);
    preprocess(s);
}

// Model::generateCUDATextures (Model.cpp:350-389): level 0 aliases the filtered depth.
// The mask pyramid of the reference is dead (N10) and not built.
void MaskFusion::generateCUDATextures(cudaStream_t s)
{
    const float* d[3] = {depthFilt, depthPyr[1].p, depthPyr[2].p};
    float4* v3[3] = {vmap[0].p, vmap[1].p, vmap[2].p};
    float4* n3[3] = {nmap[0].p, nmap[1].p, nmap[2].p};
    launch_pyrdown2_f(depthFilt, W, H, depthPyr[1], depthPyr[2], on(s));
    launch_vmap_nmap3(d, W, H, cam, cfg.depthCutoff, v3, n3, on(s));
    frameMapsValid = true;
}

// frame side of RGBDOdometry::initRGB (RGBDOdometry.cpp:212-215): intensity pyramid, Sobel derivatives, photometric validity; shared by all models
void MaskFusion::frameIntensity(cudaStream_t s)
{
    const bool rgbTerm = cfg.rgbOnly || cfg.icpWeight < 100;
    launch_intensity(rgb, P, nextImage[0], on(s));
    launch_pyrdown2_u8(nextImage[0], W, H, nextImage[1], nextImage[2], on(s));
    if (rgbTerm) {
        const uint8_t* i3[3] = {nextImage[0].p, nextImage[1].p, nextImage[2].p};
        short2* g3[3] = {nextGrad[0].p, nextGrad[1].p, nextGrad[2].p};
        uint8_t* r3[3] = {rgbValid[0].p, rgbValid[1].p, rgbValid[2].p};
        launch_sobel3(i3, W, H, g3, r3, on(s));
    }
    intensityValid = true;
}

// Model::performTracking for a batch of models: one launch sequence, blockIdx.y = model.
// viaResult: the multi-model schedule reads the tracked poses back inside the frame's FrameResult (applyFrameResult) instead of the
// -static path's dedicated copy behind the tracking kernel.
void MaskFusion::trackModels(const std::vector<Model*>& ms, bool viaResult)
{
    if (ms.empty()) return;
    if ((int)ms.size() > TRACK_MAX_JOBS) throw CudaError{"too many tracked models for one batch"};
    const bool rgbTerm = cfg.rgbOnly || cfg.icpWeight < 100;
    if (!frameMapsValid) generateCUDATextures();
    if ((rgbTerm || cfg.so3) && !intensityValid) frameIntensity();
    unsigned lightMask = 0;          // jobs with a validity bitmask (object models): small share of the tracker's grid
    for (size_t j = 0; j < ms.size(); ++j) {
        Model* m = ms[j];
        if (!viaResult) m->lastPose = m->pose;                       // Model.cpp:430 (multi-model: applied with the result)
        m->prepareTracking();
        TrackJob& J = hJobs[j];
        for (int l = 0; l < 3; ++l) {
            J.vmapC[l] = vmap[l]; J.nmapC[l] = nmap[l]; J.nextImage[l] = nextImage[l]; J.nextGrad[l] = nextGrad[l]; J.rgbValid[l] = rgbValid[l];
            J.vmapG[l] = m->vmapG[l]; J.nmapG[l] = m->nmapG[l]; J.lastDepth[l] = m->lastDepth[l]; J.lastImage[l] = m->lastImage[l];
            J.cloud[l] = m->cloud[l]; J.corres[l] = m->corres[l];
        }
        J.lastNextImage2 = m->lastNextImage2; J.st = m->trackState; J.partial = m->partial;
        J.dpose = m->dpose;
        for (int l = 0; l < 3; ++l) J.validBits[l] = m->validBits[l].p;
        if (J.validBits[0] != nullptr) lightMask |= 1u << j;
    }
    if (preWaitPending) {            // the frame's preprocessing ran on preStream: the tracker is the first consumer on the main stream
        cudaCheck(cudaStreamWaitEvent(stream, preDone, 0), "cudaStreamWaitEvent");
        preWaitPending = false;
    }
    on().mark("copy_jobs");
    // hJobs is reused every frame: the next frameBegin first waits (finalisePending) for an event recorded behind this copy
    cudaCheck(cudaMemcpyAsync(dJobs, hJobs, ms.size() * sizeof(TrackJob), cudaMemcpyHostToDevice, stream), "jobs upload");
    if ((++trackEpoch << 6) == 0u) ++trackEpoch;                     // flag 0 = "never written"
    launch_tracking(dJobs, (int)ms.size(), W, H, cam, cfg.rgbOnly != 0, cfg.icpWeight, cfg.pyramid != 0, cfg.fastOdom != 0, cfg.so3 != 0, trackEpoch,
                    on(), lightMask);
    on().mark("copy_pose_d2h");
    for (Model* m : ms) {
        if (!viaResult)
            cudaCheck(cudaMemcpyAsync(m->hTrackOut, (const char*)m->trackState.p + offsetof(TrackState, out), 40 * sizeof(float),
                                      cudaMemcpyDeviceToHost, stream), "pose D2H");
        if (cfg.so3)   // std::swap(lastNextImage, nextImage) (RGBDOdometry.cpp:484-488): only level 2 is ever read
            cudaCheck(cudaMemcpyAsync(m->lastNextImage2, nextImage[2], (size_t)(W >> 2) * (H >> 2), cudaMemcpyDeviceToDevice, stream), "so3 swap");
    }
    if (viaResult) return;
    cudaCheck(cudaEventRecord(trackDone, stream), "cudaEventRecord");
    pendingModels = ms; pendingTrack = true;
}

// host copies of the tracked poses (and, multi-model, of everything else a frame decides): waits for an event that lies MID-frame
// (behind the tracking kernel / the vote kernel), not for the rest of the frame
void MaskFusion::finalisePending()
{
    if (pendingTrack) {
        cudaCheck(cudaEventSynchronize(trackDone), "cudaEventSynchronize");
        for (Model* m : pendingModels) {
            memcpy(m->pose.m, m->hTrackOut, 16 * sizeof(float));
            memcpy(m->lastTransform.m, m->hTrackOut + 16, 16 * sizeof(float));
        }
        pendingTrack = false; pendingModels.clear();
    }
    if (pendingResult) applyFrameResult();
    if (pendingLog) { pendingLog = false; logPoses(pendingTimestamp); }
}

// MaskFusion.cpp:577-592: one pose-log entry per model per frame
void MaskFusion::logPoses(int64_t timestamp)
{
    Model* g = models[0].get();
    for (size_t i = 0; i < models.size(); ++i) {
        Model* m = models[i].get();
        Mat4 T = (i == 0) ? g->pose : mul(g->pose, rigidInverse(m->pose));     // MaskFusion.cpp:581-583
        float R[9] = {T.m[0], T.m[1], T.m[2], T.m[4], T.m[5], T.m[6], T.m[8], T.m[9], T.m[10]}, q[4];
        rotToQuat(R, q);
        double e[8] = {(double)timestamp, T.m[3], T.m[7], T.m[11], q[0], q[1], q[2], q[3]};
        m->poseLog.insert(m->poseLog.end(), e, e + 8);
    }
}

void MaskFusion::predict()
{
    for (auto& m : models) if (m->owned) m->combinedPredict(cfg.maxDepthProcessed, tick, tick, cfg.timeDelta);   // MaskFusion.cpp:616-628
}

// GlobalProjection::project (GlobalProjection.cpp:43-107): all models into one depth-tested key image; the key's low word
// is (model list index << 26 | surfel id), i.e. the reference's draw order.  The ID image stays on the device.
void MaskFusion::globalProjection() { segTables(segModels()); projectLocal(); projectResolve(); }

void MaskFusion::checkModelCount() const
{
    if (models.size() > MF_MAX_MODELS - 1) throw CudaError{"global projection / segmentation support up to 63 models"};
}

// the model list as segmentation sees it: list order, ids, classes and the id a new model would take
SegModels MaskFusion::segModels()
{
    checkModelCount();
    SegModels sm; memset(&sm, 0, sizeof sm);
    sm.n = (int)models.size();
    for (int i = 0; i < sm.n; ++i) { sm.id[i] = models[i]->id; sm.classID[i] = models[i]->classID; }
    sm.nextID = getNextModelID(false);
    return sm;
}

// id <-> list-index tables of a model list, as a kernel argument (no staging buffer, no synchronisation)
void MaskFusion::segTables(const SegModels& sm)
{
    SegTables t; memset(&t, 0, sizeof t);
    for (int i = 0; i < sm.n; ++i) { t.idToIndex[sm.id[i]] = (uint8_t)i; t.indexToId[i] = sm.id[i]; t.isModel[sm.id[i]] = 1; }
    launch_seg_tables(t, tblIdToIndex, tblIndexToId, tblIsModel, on());
}

// local half: every model whose surfels live here goes into the key image (ghost models arrive through the min all-reduce)
void MaskFusion::projectLocal()
{
    checkModelCount();
    for (size_t i = 0; i < models.size(); ++i) {
        Model* m = models[i].get();
        if (!m->owned) continue;
        launch_splat_project_only(m->current(), m->dCount(), m->dpose, cam, W, H, cfg.depthCutoff, 12.0f /* :61 */, tick, tick,
                                  cfg.timeDelta, (uint32_t)i << 26, rayTab, projKeys, on(), m->capacity);
    }
}

void MaskFusion::projectResolve()
{
    launch_proj_resolve(projKeys, P, tblIndexToId, projectedIDs, on());
}

// edge-ness -> threshold -> close -> invert (MfSegmentation.cpp:149-208)
void MaskFusion::edgeMaps()
{
    if (!frameMapsValid) generateCUDATextures();
    launch_geometric_edges(vmap[0], nmap[0], W, H, cfg.segWeightDistance, cfg.segWeightConvexity, cfg.segThreshold, edgeMap, edgeBinary, on());
    launch_morph_close_invert(edgeBinary, edgeBuf, W, H, cfg.segMorphEdgeRadius, cfg.segMorphEdgeIterations, edgeInv, on());
}

// MfSegmentation::performSegmentation (MfSegmentation.cpp:83-538) with the CPU tail on the GPU (mf_seg.cu) and NO host round trip:
// the number of components, the number of masks and their classes are read by the kernels from device memory; the mask -> model vote
// (:433-492) is a kernel; its decision (new label?) travels to the host inside the FrameResult and is applied by applyFrameResult().
void MaskFusion::performSegmentation(const SegModels& sm, bool allowNew)
{
    edgeMaps();
    // the first readers of the frame's mask and of the header's mask fields: a detector's hand-off must have landed (tracking and the ID
    // projection above ran next to the detector)
    waitHandoff(stream);
    if (maskCommPending) { cudaCheck(cudaStreamWaitEvent(stream, evComm, 0), "cudaStreamWaitEvent"); maskCommPending = false; }   // sharded: the masks' broadcast
    segmentEdges(sm, allowNew, mask);                       // writes textureMask directly (:297)
}

// everything of performSegmentation after the edge map (:221-522), on the inverted edge map (edgeInv), the frame's raw depth, mask and
// header, and the projected-ID image, for the model list `sm` (whose tables segTables(sm) has set); the segmentation goes to `out`, the
// vote's decision to dRes.  The ignore map and maskToID persist across calls like the members of the reference class.
void MaskFusion::segmentEdges(const SegModels& sm, bool allowNew, uint8_t* out)
{
    const int nModels = sm.n;
    const Enq q = on();
    // ignore map (:221-235)
    launch_person_table(dHdr, personClassID, tblIsPerson, q);
    launch_apply_ignore(frameMask, tblIsPerson, dHdr, P, ignoreMap, edgeInv, q);
    // connected components + 5 edge-removal sweeps (:238-291)
    launch_cc(edgeInv, W, H, ccL, ccDense, ccLabA, ccArea, ccBox, ccCounter, q);
    launch_remove_edges(ccLabA, ccLabB, depthRaw, ccArea, W, H, 5, q);
    int* lab = ccLabB;                                     // odd number of sweeps ends in B
    // overlap histograms (:303-346)
    launch_clear_hist(ccCounter, dHdr, nModels, compModel, compMask, q);
    maskPixels.zero(stream);
    launch_seg_hist(lab, projectedIDs, frameMask, P, tblIdToIndex, nModels, dHdr, compModel, compMask, q);
    launch_component_map(ccCounter, ccArea, compModel, compMask, nModels, dHdr, tblIndexToId, minMappedComponentSize, mapToMask, absorbId, maskPixels, q);
    launch_seg_assign(lab, mapToMask, ignoreMap, P, segTmp, q);
    // closing of the mask-id image with an elliptic element (:424-426, inside `if (nMasks)`); edgeBuf is free again at this point
    launch_morph_close_ellipse(segTmp, edgeBuf, W, H, cfg.segMorphMaskRadius, cfg.segMorphMaskIterations, dHdr, q);
    // mask -> model vote (:433-492)
    cudaCheck(cudaMemsetAsync(maskOverlap, 0, (size_t)nModels * 256 * sizeof(unsigned), stream), "memset");
    launch_mask_overlap(segTmp, projectedIDs, tblIdToIndex, tblIsModel, P, maskOverlap, q);
    VoteParams vp; memset(&vp, 0, sizeof vp);
    vp.nModels = nModels; vp.allowNew = allowNew ? 1 : 0; vp.personClassID = personClassID;
    vp.minNew = (unsigned)(size_t)(cfg.minRelSizeNew * (size_t)P); vp.maxNew = (unsigned)(size_t)(cfg.maxRelSizeNew * (size_t)P);
    vp.minMaskModelOverlap = minMaskModelOverlap; vp.nextModelID = sm.nextID;
    for (int i = 0; i < nModels; ++i) { vp.modelClass[i] = sm.classID[i]; vp.modelID[i] = sm.id[i]; }
    launch_vote(dHdr, vp, maskPixels, maskOverlap, ccCounter, tblMaskToID, dRes, q);
    launch_seg_final(segTmp, lab, mapToMask, absorbId, tblMaskToID, ccBox, P, W, out, q);
}

// MaskFusion::getNextModelID (MaskFusion.cpp:712-730)
unsigned char MaskFusion::getNextModelID(bool assign)
{
    unsigned char next = nextID;
    if (assign) {
        if (models.size() == 256) throw CudaError{"getNextModelID(): maximum amount of models is already in use (256)"};
        while (true) {
            nextID++;
            bool occupied = false;
            for (auto& m : models) if (nextID == m->id) occupied = true;
            if (!occupied) break;
        }
    }
    return next;
}

// model->getFrameOdometry().initFirstRGB(textureRGB): the frame's intensity pyramid (built here unless it is current); its level 2 is
// the model's first lastNextImage
void MaskFusion::initFirstRGB(Model* m)
{
    if (!intensityValid) {
        launch_intensity(rgb, P, nextImage[0], on());
        launch_pyrdown2_u8(nextImage[0], W, H, nextImage[1], nextImage[2], on());
    }
    cudaCheck(cudaMemcpyAsync(m->lastNextImage2, nextImage[2], (size_t)(W >> 2) * (H >> 2), cudaMemcpyDeviceToDevice, stream), "initFirstRGB");
}

// MaskFusion::spawnObjectModel + moveNewModelToList (MaskFusion.cpp:671-690)
Model* MaskFusion::spawnObjectModel()
{
    Model* g = models[0].get();
    // sharded mode: the new store goes to the least-loaded rank; every rank evaluates the same rule on the same replicated list
    int64_t loads[64] = {0};
    // load of a rank = (number of models it tracks, their surfel capacity): every tracked model walks the whole image in the tracker, so
    // the model count dominates; the capacity breaks ties (the background's store is the big one)
    for (auto& m : models) loads[m->ownerRank] += ((int64_t)1 << 32) + m->capacity;
    if (detRank >= 0) loads[detRank] += (int64_t)1 << 32;          // the network weighs like one more tracked model there
    const int ownerRank = world > 1 ? pickOwner(loads, world) : 0;
    models.emplace_back(new Model(this, getNextModelID(true), cfg.confObject, false, cfg.capacityObject, ownerRank, ownerRank != rank));
    Model* nm = models.back().get();
    if (nm->owned) { initFirstRGB(nm); intensityValid = true; }
    nm->makeStatic(g->pose);
    return nm;
}

int MaskFusion::pickOwner(const int64_t* loads, int world)
{
    int best = 0;
    for (int r = 1; r < world; ++r) if (loads[r] <= loads[best]) best = r;
    return best;
}

void MaskFusion::configureShard(int rank_, int world_)
{
    if (world_ < 1 || world_ > 64 || rank_ < 0 || rank_ >= world_) throw CudaError{"configureShard: need 0 <= rank < world <= 64"};
    if (detector || detRank >= 0)
        throw CudaError{"configureShard: a detector is attached; detach it, configure the shards, then attach it with mf_shard_attach_detector"};
    if (tick != 1) throw CudaError{"configureShard: must be called before the first frame"};
    if (queueLength > 1) throw CudaError{"configureShard: a frame queue is set (mf_set_frame_queue); the sharded mode runs without one"};
    if (world_ > 1 && !cfg.enableMultipleModels) throw CudaError{"configureShard: a -static run has one model and does not shard (run replicas instead)"};
    rank = rank_; world = world_;
    if (rank != 0) {          // the background model lives on rank 0
        Model* g = models[0].get();
        models[0].reset(new Model(this, g->id, cfg.confGlobal, true, cfg.capacityGlobal, 0, true));
        sync();
    }
}

// communicator of the shards (mf_shard_comm_init): from here on the three exchanges of a frame are NCCL calls on the context's stream
void MaskFusion::initShardComm(const unsigned char* id128, int rank_, int world_)
{
    if (!cfg.enableMultipleModels) throw CudaError{"initShardComm: a -static run has one model and does not shard (run replicas instead)"};
    if (queueLength > 1) throw CudaError{"initShardComm: a frame queue is set (mf_set_frame_queue); the sharded mode runs without one"};
    if (detector && detRank < 0)
        throw CudaError{"initShardComm: a detector is attached to this single process; detach it, then attach it to the shards with mf_shard_attach_detector"};
    if (world == 1 && world_ > 1) configureShard(rank_, world_);
    if (rank_ != rank || world_ != world) throw CudaError{"initShardComm: rank / world differ from configureShard"};
    cudaCheck(cudaSetDevice(device), "cudaSetDevice");
    shard.init(id128, rank_, world_);
    shardNccl = true;
}

// after the entry point's own checks: a backbone, or (asDetector) a detector on some rank of the run; `det` is its handle where it runs
void MaskFusion::attachNetwork(const char* who, bool asDetector, mf_detector* det)
{
    if (asDetector && backbone)
        throw CudaError{std::string(who) + ": a backbone is attached (the detector runs its own backbone on the same stream); detach it first"};
    if (!asDetector && (detector || detRank >= 0))
        throw CudaError{std::string(who) + ": a detector is attached (it runs its own backbone on the same stream); detach it first"};
    waitNetwork();
    if (det) detector_reserve_image(det, W, H);
    if (!netRGBA.p) netRGBA.alloc(P);
}

void MaskFusion::attachBackbone(mf_backbone* bb, int everyK)
{
    if (bb) {
        if (!cfg.enableMultipleModels) throw CudaError{"attachBackbone: a -static context runs no segmentation to feed"};
        attachNetwork("attachBackbone", false, nullptr);
    }
    backbone = bb; backboneEvery = bb ? (everyK > 0 ? everyK : 1) : 0;
}

void MaskFusion::attachDetector(mf_detector* det, int everyK)
{
    if (det) {
        if (!cfg.enableMultipleModels) throw CudaError{"attachDetector: a -static context runs no segmentation to feed"};
        if (world > 1 || shardNccl) throw CudaError{"attachDetector: this context is one rank of an object-sharded run; attach the detector on every rank with mf_shard_attach_detector"};
        attachNetwork("attachDetector", true, det);
    } else
        waitNetwork();
    detector = det; detectorEvery = det ? (everyK > 0 ? everyK : 1) : 0;
}

void MaskFusion::waitNetwork()
{
    for (auto& f : ring) if (f->netUsed) cudaCheck(cudaEventSynchronize(f->netDone), "cudaEventSynchronize");
}

// every rank of a sharded run, between the same frames, with the same everyK / detectorRank; det on detectorRank only.
// (NULL, 0, -1) detaches on every rank.
void MaskFusion::attachShardDetector(mf_detector* det, int everyK, int detectorRank)
{
    if (!det && everyK == 0 && detectorRank == -1) {
        if (detRank < 0) return;
        waitNetwork();
        detector = nullptr; detectorEvery = 0; detRank = -1;
        return;
    }
    if (!cfg.enableMultipleModels) throw CudaError{"shard_attach_detector: a -static context runs no segmentation to feed"};
    if (world == 1) throw CudaError{"shard_attach_detector: not a sharded context (world == 1); call mf_shard_configure or mf_shard_comm_init first, or use mf_attach_detector for one process"};
    if (detectorRank < 0 || detectorRank >= world)
        throw CudaError{"shard_attach_detector: detector_rank " + std::to_string(detectorRank) + " outside [0, " + std::to_string(world) + ")"};
    if (det && rank != detectorRank)
        throw CudaError{"shard_attach_detector: a detector was given on rank " + std::to_string(rank) + ", which is not the detector rank " + std::to_string(detectorRank)};
    if (!det && rank == detectorRank) throw CudaError{"shard_attach_detector: no detector given on the detector rank " + std::to_string(detectorRank)};
    attachNetwork("shard_attach_detector", true, det);
    detector = det; detectorEvery = everyK > 0 ? everyK : 1; detRank = detectorRank;
}

void MaskFusion::waitHandoff(cudaStream_t s)
{
    FrameSlot& f = *ring[curSlot];
    if (!f.handoff) return;
    cudaCheck(cudaStreamWaitEvent(s, f.netDone, 0), "cudaStreamWaitEvent");
    f.handoff = false;
}

// external transport (no communicator), between frameProject and frameEnd: on a mask-exchange frame, the detector rank's stream first
// waits for the hand-off; the caller then broadcasts [frameMask, +P + sizeof(FrameHdr)) from detRank.  With a communicator the library
// issues that broadcast itself, and there is nothing for the caller to move.
bool MaskFusion::shardFrameMasks(void** ptr, size_t* bytes)
{
    if (shardNccl || !fExchange) return false;
    waitHandoff(stream);
    *ptr = frameMask; *bytes = (size_t)P + sizeof(FrameHdr);
    return true;
}

// On the network's stream behind the frame's upload (slot `uploaded`, which covers the header with nMasks = 0); the host never waits.
// The RGBA copy the network reads is made on that stream too, so consecutive frames share it without further events.
// Backbone: RGBA image -> letter-boxed network input -> ResNet-101-FPN forward.  Detector (MfSegmentation.cpp:128-131: `if
// (frame->mask.total() == 0) maskRCNN->executeSequential(frame)`): detection of the RGBA copy, then the hand-off into the mask and
// header of the frame's slot.  The RGBA copy belongs to the network's work: it is not counted in the context's launches.
void MaskFusion::runNetwork(int slot, bool runBackbone)
{
    FrameSlot& f = *ring[slot];
    cudaStream_t ns = runBackbone ? backbone_stream(backbone) : detector_stream(detector);
    cudaCheck(cudaStreamWaitEvent(ns, f.uploaded, 0), "cudaStreamWaitEvent");
    launch_unpack_rgb(f.packet.p, netRGBA, P, Enq{ns, nullptr});
    if (runBackbone) {
        backbone_mold(backbone, netRGBA, W, H);
        cudaCheck(cudaEventRecord(f.netDone, ns), "cudaEventRecord");               // the slot is free again once the input is molded
        f.netUsed = true;
        backbone_forward(backbone, backbone_input(backbone));
    } else {
        detector_detect(detector, netRGBA, W, H);
        detector_frame_masks(detector, slotMask(slot), slotHdr(slot));
        // one event for both guards: the slot may be reused, and its mask / header are written
        cudaCheck(cudaEventRecord(f.netDone, ns), "cudaEventRecord");
        f.netUsed = true; f.handoff = true;
    }
}

void MaskFusion::waitMain(cudaStream_t s)
{
    cudaCheck(cudaEventRecord(evMain, stream), "cudaEventRecord");
    cudaCheck(cudaStreamWaitEvent(s, evMain, 0), "cudaStreamWaitEvent");
}

// commOnPre (a communicator on an overlapped frame): every collective runs on preStream, one stream per communicator, so their order is
// the same on every rank by construction.  Collectives issued back to back share one commStream().  Otherwise they run on the main stream.
cudaStream_t MaskFusion::commStream()
{
    if (!commOnPre) return stream;
    waitMain(preStream);
    return preStream;
}

void MaskFusion::joinComm(bool now)
{
    if (!commOnPre) return;
    cudaCheck(cudaEventRecord(evComm, preStream), "cudaEventRecord");
    if (now) cudaCheck(cudaStreamWaitEvent(stream, evComm, 0), "cudaStreamWaitEvent");
    else maskCommPending = true;
}

// the models of the frame in flight as the lifecycle kernels see them
LifeParams MaskFusion::lifeParams() const
{
    LifeParams lp; memset(&lp, 0, sizeof lp);
    if (models.size() > MF_MAX_MODELS) throw CudaError{"more than 64 models"};
    lp.nModels = (int)models.size(); lp.rank = rank;
    for (size_t i = 0; i < models.size(); ++i) {
        const Model* m = models[i].get();
        LifeModel& L = lp.m[i];
        L.tracked = m->tracked ? 1 : 0; L.owned = m->owned ? 1 : 0; L.ownerRank = m->ownerRank;
        if (m->owned) {
            L.dpose = m->dpose.p; L.count = m->dCount();
            L.trackOut = reinterpret_cast<const float*>(reinterpret_cast<const char*>(m->trackState.p) + offsetof(TrackState, out));
        }
        memcpy(L.initialC2Winv, m->initialC2Winv.m, sizeof L.initialC2Winv);
    }
    return lp;
}

// external transport (no NCCL communicator): this rank's rows to the host / the gathered rows of all ranks back to the device
void MaskFusion::getShardPoses(float* out)
{
    cudaCheck(cudaMemcpyAsync(out, poseTable.p, (size_t)MF_MAX_MODELS * 32 * sizeof(float), cudaMemcpyDeviceToHost, stream), "rows D2H");
    cudaCheck(cudaStreamSynchronize(stream), "cudaStreamSynchronize");
}
void MaskFusion::setShardPoses(const float* all)
{
    cudaCheck(cudaMemcpyAsync(gathered.p, all, (size_t)world * MF_MAX_MODELS * 32 * sizeof(float), cudaMemcpyHostToDevice, stream), "rows H2D");
    cudaCheck(cudaStreamSynchronize(stream), "cudaStreamSynchronize");
}

bool MaskFusion::processFrame(const uint8_t* rgbIn, const float* depthIn, int64_t timestamp, const uint8_t* maskIn, const Mat4* inPose,
                              float weightMultiplier, bool bootstrap, bool onDevice)
{
    if (world > 1 && !shardNccl) throw CudaError{"processFrame: this context is one shard of several without a communicator; call mf_shard_comm_init, or drive the frame_begin/project/end phases and move the rows / keys yourself"};
    if (frameBegin(rgbIn, depthIn, timestamp, maskIn, inPose, bootstrap, onDevice)) {
        frameProject();
        frameEnd(weightMultiplier);
    }
    if (copyPending) {               // the caller's host buffers are free again on return, as with the reference's synchronous upload
        cudaCheck(cudaEventSynchronize(inputsCopied), "cudaEventSynchronize");
        copyPending = false;
    }
    return false;
}

// MaskFusion.cpp:200-209: the call's frame joins the queue; once queueLength frames wait, the oldest one is processed (MaskFusion.cpp:
// 210-276 from here: filter, first-frame initialisation or tracking of every model whose store lives here).  inPose, bootstrap and (in
// frameEnd) weightMultiplier belong to the call and apply to the frame it processes, as in the reference.
bool MaskFusion::frameBegin(const uint8_t* rgbIn, const float* depthIn, int64_t timestamp, const uint8_t* maskIn, const Mat4* inPose, bool bootstrap,
                            bool onDevice)
{
    const bool multi = cfg.enableMultipleModels != 0;
    if (world > 1 && inPose) throw CudaError{"sharded mode tracks every frame (no external poses)"};
    if (multi && bootstrap && inPose) throw CudaError{"bootstrap poses are supported by the -static schedule only"};
    finalisePending();                                  // previous frame: tracked poses, pose log, (multi) inactivations and the deferred spawn
    const int q = queued;                               // frames pushed by earlier calls and not processed yet
    const bool process = q + 1 >= (queueLength > 1 ? queueLength : 1);
    const int ptick = tick + q;                         // the tick the pushed frame is processed at: the n-th call's frame at tick n
    const bool tracking = process && tick > 1 && (bootstrap || !inPose);
    fExchange = detRank >= 0 && multi && tracking && tick % detectorEvery == 0;    // sharded: no queue, ptick == tick
    // Detection is decided when the frame is pushed, for the tick it is processed at.  One process: the caller's mask decides on the
    // host; without a queue the pushing call is the processing call, and an in_pose frame does not segment.  A queued frame cannot know
    // whether the call that pops it passes an in_pose: if it does, the frame does not segment and its detection goes unused.  Sharded: the
    // detector rank detects on every exchange frame and k_frame_masks keeps a caller's mask (FrameHdr::maskGiven), which only rank 0 has seen.
    const bool detWanted = detRank >= 0 ? fExchange : multi && !maskIn && ptick > 1 && (q > 0 || bootstrap || !inPose);
    // Overlapped tracking frames (pre): upload + bilateral + pyramids + maps + intensity/Sobel of THIS frame go to preStream and into the
    // other image set, so they run next to the previous frame's fusion / clean / prediction tail still queued on the main stream (that
    // tail reads the previous frame's images; the copy engine and the issue-bound bilateral overlap well with the HBM-bound
    // clean/scatter).  The maps need no further events: finalisePending() above has waited for the previous frame's tracker, their last
    // reader.  A shard overlaps only with a communicator, which then runs every collective of the frame on preStream (commStream).
    // A -static context never shards (configureShard, initShardComm).
    const bool pre = tracking && !rec.prof.on && (world == 1 || shardNccl);
    cudaStream_t s = pre ? preStream : stream;
    commOnPre = pre && multi && shardNccl;
    // the spawn that finalisePending() just carried out reads the previous frame's intensity pyramid (initFirstRGB), which this frame's
    // preprocessing overwrites: on such (rare) frames the preprocessing waits for the main stream
    if (spawnedInApply && pre) waitMain(s);
    spawnedInApply = false;
    // the slot the push writes and the image set this frame's preprocessing writes were last read by frames processed before the last pop
    if (s != stream && retiredValid) cudaCheck(cudaStreamWaitEvent(s, retired, 0), "cudaStreamWaitEvent");
    pushFrame(rgbIn, depthIn, timestamp, maskIn, onDevice, s, ptick, detWanted);
    if (!process) return false;
    popFrame(s);
    fTimestamp = ring[curSlot]->timestamp; fHasPose = inPose != nullptr; if (inPose) fInPose = *inPose; fBootstrap = bootstrap;
    preprocess(s);
    if (pre) {
        generateCUDATextures(s);
        if (cfg.rgbOnly || cfg.icpWeight < 100 || cfg.so3) frameIntensity(s);
        cudaCheck(cudaEventRecord(preDone, s), "cudaEventRecord");
        preWaitPending = true;
    }
    Model* g = models[0].get();
    fTracked = false;
    for (auto& m : models) m->tracked = false;
    if (tick == 1) {
        if (g->owned) {
            g->initialise(tick);
            initFirstRGB(g);                            // globalModel->getFrameOdometry().initFirstRGB (MaskFusion.cpp:238)
        }
    } else if (tracking) {
        if (!frameMapsValid) generateCUDATextures();
        // MaskFusion.cpp:247-276: the global model and every tracked object share one batched launch sequence
        std::vector<Model*> tracked;
        for (size_t i = 0; i < models.size(); ++i) {
            Model* m = models[i].get();
            m->tracked = (i == 0 || m->nonstatic || cfg.trackAllModels);
            if (m->owned && m->tracked) tracked.push_back(m);
        }
        trackModels(tracked, multi);
        if (preWaitPending) {            // no model is tracked here (a shard without stores): the later passes still read this frame's maps
            cudaCheck(cudaStreamWaitEvent(stream, preDone, 0), "cudaStreamWaitEvent");
            preWaitPending = false;
        }
        fTracked = true;
        if (multi) {
            // pose rows of the models tracked here; with a communicator every rank receives every rank's rows (all-gather)
            launch_pack_rows(lifeParams(), poseTable, on());
            if (shardNccl) {
                on().mark("nccl_allgather_poses");
                shard.allGatherFloats(poseTable, gathered, (size_t)MF_MAX_MODELS * 32, commStream());
                joinComm(true);
            }
        } else if (bootstrap && inPose) finalisePending();     // -static bootstrap: the host composes the tracked pose with the given one
    }
    return true;
}

// the frame joins the queue: its packet goes into the next free slot on `s`, and the attached network runs on it now (MaskRCNN.cpp:
// 183-200 writes masks into queued frames)
void MaskFusion::pushFrame(const uint8_t* rgbIn, const float* depthIn, int64_t timestamp, const uint8_t* maskIn, bool onDevice, cudaStream_t s,
                           int ptick, bool detWanted)
{
    const int k = (curSlot + queued + 1) % (int)ring.size();
    FrameSlot& f = *ring[k];
    if (f.netUsed) cudaCheck(cudaStreamWaitEvent(s, f.netDone, 0), "cudaStreamWaitEvent");   // an older frame's network read the slot
    if (shardNccl) {
        // object-sharded: rank 0 holds the loader; the frame packet (images + mask + header, one buffer) goes to every rank over NVLink
        if (rank == 0) uploadInputs(k, rgbIn, depthIn, maskIn, timestamp, onDevice, s);
        on(s).mark("nccl_broadcast_packet");
        shard.broadcast(f.packet.p, packetBytes(), 0, s);
    } else
        uploadInputs(k, rgbIn, depthIn, maskIn, timestamp, onDevice, s);     // -static: textureMask stays all zero (MaskFusion.cpp:223-230)
    f.timestamp = timestamp; f.upStream = s; f.handoff = false;
    const bool runBackbone = backbone && ptick % backboneEvery == 0, runDetector = detector && detWanted && ptick % detectorEvery == 0;
    if (runBackbone || runDetector || queueLength > 1) cudaCheck(cudaEventRecord(f.uploaded, s), "cudaEventRecord");
    queued++;
    if (runBackbone || runDetector) runNetwork(k, runBackbone);
}

// the oldest queued frame becomes the current one.  The frame processed before it keeps its slot and its image set.
void MaskFusion::popFrame(cudaStream_t s)
{
    cudaCheck(cudaEventRecord(retired, stream), "cudaEventRecord");
    retiredValid = true;
    const int k = (curSlot + 1) % (int)ring.size();
    queued--;
    selectSlot(k);
    selectSet(curSet ^ 1);
    FrameSlot& f = *ring[k];
    if (f.upStream != s) cudaCheck(cudaStreamWaitEvent(s, f.uploaded, 0), "cudaStreamWaitEvent");
}

// MaskFusion.cpp:257-290 after the poses are known everywhere: inactivation, static poses (device side), local part of the ID projection
void MaskFusion::frameProject()
{
    if (!fTracked) return;
    if (!cfg.enableMultipleModels) {
        if (fBootstrap && fHasPose) { Model* g = models[0].get(); g->overridePose(mul(g->pose, fInPose)); }
        return;
    }
    launch_lifecycle(lifeParams(), world > 1 ? gathered.p : poseTable.p, dRes, on());
    projectLocal();                                                            // :289-290
}

// MaskFusion.cpp:290-607: segmentation (replicated: every rank holds the same merged key image), fusion of the local stores, prediction
void MaskFusion::frameEnd(float weightMultiplier)
{
    const bool multi = cfg.enableMultipleModels != 0;
    Model* g = models[0].get();
    fWeight = weightMultiplier;
    if (tick > 1) {
        if (fTracked) {
            if (multi) {
                if (shardNccl) {
                    on().mark("nccl_allreduce_keys");
                    cudaStream_t cs = commStream();
                    shard.allReduceMinU64(projKeys, (size_t)P, cs);
                    joinComm(true);
                    if (fExchange) {
                        // detector frame: the detector rank's mask and header replace every rank's (a caller's mask travels back unchanged).
                        // The main stream waits for it only where segmentation first reads the mask.
                        on().mark("nccl_broadcast_masks");
                        waitHandoff(cs);
                        shard.broadcast(frameMask, (size_t)P + sizeof(FrameHdr), detRank, cs);
                        joinComm(false);
                    }
                }
                const SegModels sm = segModels();
                segTables(sm);
                projectResolve();
                if (spawnOffset < cfg.modelSpawnOffset) spawnOffset++;
                performSegmentation(sm, spawnOffset >= cfg.modelSpawnOffset);
                // what the host needs from this frame, in one copy behind the vote kernel; picked up by the next finalisePending()
                on().mark("copy_result_d2h");
                cudaCheck(cudaMemcpyAsync(hRes, dRes.p, sizeof(FrameResult), cudaMemcpyDeviceToHost, stream), "result D2H");
                cudaCheck(cudaEventRecord(resEvt, stream), "cudaEventRecord");
                pendingResult = true;
                for (size_t i = 1; i < models.size(); ++i) models[i]->maxDepth = 30.0f + 30.0f * 1.2f;   // getMaxDepth(30, 30), :292,337-341
                for (size_t i = 1; i < models.size(); ++i) {                           // :369-374
                    float f = (float)models[i]->age / 25.0f;
                    models[i]->confidenceThreshold = f < 4.5f ? f : 4.5f;
                }
            }
        } else {
            g->overridePose(fInPose);
        }
        if (!cfg.rgbOnly) {
            for (auto& m : models) if (m->owned) m->predictIndices(tick, cfg.maxDepthProcessed, cfg.timeDelta, false);
            for (auto& m : models) if (m->owned) m->fuse(tick, cfg.depthCutoff, weightMultiplier);
            for (auto& m : models) if (m->owned) m->predictIndices(tick, cfg.maxDepthProcessed, cfg.timeDelta);
            for (auto& m : models) if (m->owned) m->clean(tick, cfg.timeDelta, cfg.maxDepthProcessed);
        }
    }
    predict();          // MaskFusion.cpp:569 (the call at :423 is dead in open-loop mode: its outputs are overwritten here)
    fTick = tick;
    tick++;
    if (pendingResult) { /* the pose-log entry is written by applyFrameResult, after the spawn it may carry out */ }
    else if (pendingTrack) { pendingLog = true; pendingTimestamp = fTimestamp; }    // -static: the entry is written when the pose arrives
    else logPoses(fTimestamp);
    for (auto& m : models) m->age++;
}

// Everything the host learns from a multi-model frame, applied at the start of the next one (or by any query in between), in the
// order of the reference's frame: tracked poses (Model.cpp:427-447) -> inactivation (MaskFusion.cpp:268-272, 699-713) -> spawn of the
// model MfSegmentation asked for and its first fusion FROM THAT FRAME'S DATA (:313-353; the input set, textureMask and the intensity
// pyramid of the frame are still untouched) -> pose log (:577-592).  Identical on every rank of a sharded run (replicated inputs).
void MaskFusion::applyFrameResult()
{
    cudaCheck(cudaEventSynchronize(resEvt), "cudaEventSynchronize");
    pendingResult = false;
    const FrameResult& R = *hRes;
    for (size_t i = 0; i < models.size(); ++i) {
        Model* m = models[i].get();
        if (!m->tracked && i == 0) continue;
        m->lastPose = m->pose;
        memcpy(m->pose.m, R.poses[i], 16 * sizeof(float));
        if (m->tracked) memcpy(m->lastTransform.m, R.poses[i] + 16, 16 * sizeof(float));
    }
    for (size_t i = models.size(); i-- > 1;) {
        if (!R.dead[i]) continue;
        Model* m = models[i].get();
        const unsigned cnt = m->owned ? R.deadCount[i] : modelKeepMinSurfels;
        if (!enableSmartModelDelete || (cnt >= modelKeepMinSurfels && m->confidenceThreshold > modelKeepConfThreshold)) {
            if (m->owned) launch_set_count(m->dCount(), cnt, on());                           // the store as it was when the model left
            inactiveModels.push_back(std::move(models[i]));
        }
        models.erase(models.begin() + i);
    }
    if (R.hasNewLabel) {                                                                       // :313-334
        Model* nm = spawnObjectModel();
        spawnedInApply = true;
        spawnOffset = 0;
        nm->classID = R.newClassID;
        nm->maxDepth = 30.0f + 30.0f * 1.2f;
        if (nm->owned) {                                                                       // :344-353, with the frame's own tick / weight
            const int t = fTick;
            nm->predictIndices(t, cfg.maxDepthProcessed, cfg.timeDelta);
            nm->fuse(t, cfg.maxDepthProcessed, 100.0f);
            nm->clean(t, cfg.timeDelta, cfg.maxDepthProcessed);
            nm->confidenceThreshold = 0.0f;                                                    // age 0 (:369-374)
            if (!cfg.rgbOnly) {
                nm->predictIndices(t, cfg.maxDepthProcessed, cfg.timeDelta, false);
                nm->fuse(t, cfg.depthCutoff, fWeight);
                nm->predictIndices(t, cfg.maxDepthProcessed, cfg.timeDelta);
                nm->clean(t, cfg.timeDelta, cfg.maxDepthProcessed);
            }
            nm->combinedPredict(cfg.maxDepthProcessed, t, t, cfg.timeDelta);
        }
        nm->confidenceThreshold = 0.0f;
        nm->age = 1;
    }
    logPoses(R.timestamp);
    // the frame has been processed without masks; the error surfaces here, with everything else the frame decided already applied
    if (R.detectError)
        throw CudaError{"detector: generate_id_image: special_assignments[class_id] out of range (IndexError upstream) on the frame of timestamp " +
                        std::to_string(R.timestamp) + ", which was processed without masks"};
}

}  // namespace mfb
