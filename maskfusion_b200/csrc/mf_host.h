// mf_host.h -- host classes of the H100-native dense pipeline.  Class and method names
// mirror the reference so that its call sites read the same:
//   mfb::MaskFusion  <-> MaskFusion   (Core/MaskFusion.h:47-70)
//   mfb::Model       <-> Model        (Core/Model/Model.h:128-164)
// GPUTexture* arguments of the reference become device buffers owned by these classes;
// Eigen::Matrix4f becomes Mat4 (row-major here, column-major at the C ABI).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <memory>
#include <string>
#include <vector>
#include <map>
#include "../../include/maskfusion_b200.h"
#include "mf_kernels.h"

namespace mfb {

struct Mat4 {
    float m[16];
    static Mat4 identity() { Mat4 r; for (int i = 0; i < 16; ++i) r.m[i] = (i % 5 == 0) ? 1.f : 0.f; return r; }
};
inline Mat4 rigidInverse(const Mat4& T) { Mat4 o; rigidInverse(T.m, o.m); return o; }
inline Mat4 mul(const Mat4& A, const Mat4& B) { Mat4 o; mul(A.m, B.m, o.m); return o; }
Rt toRt(const Mat4& T);

// in-stream stage timer: one CUDA event per mark; the interval up to the next mark is attributed to the mark's name.  Off by default.
struct Profiler {
    bool on = false; int used = 0;
    std::vector<Event> events; std::vector<const char*> names;     // events created with timing enabled
    std::map<std::string, std::pair<long, double>> acc;      // name -> (count, total ms)
    void resolve();
};
// what a context records about the kernels it enqueues through its Enq (MaskFusion::on)
struct LaunchRecord {
    int64_t launches = 0;               // mf_kernel_launches
    Profiler prof;
};

class MaskFusion;

// object-sharded mode: NCCL communicator of the ranks that share one replay (mf_sched.cu; libnccl is opened at run time)
struct ShardComm {
    void* comm = nullptr; int rank = 0, world = 1, version = 0; size_t bytesMoved = 0; long calls = 0;
    ShardComm() {}
    ShardComm(const ShardComm&) = delete;
    ShardComm& operator=(const ShardComm&) = delete;
    ~ShardComm();
    void init(const unsigned char* id128, int rank, int world);
    void broadcast(void* buf, size_t bytes, int root, cudaStream_t s);                               // frame packet (MaskFusion.cpp:212-217)
    void allGatherFloats(const float* send, float* recv, size_t countPerRank, cudaStream_t s);       // pose rows (MaskFusion.cpp:257-276)
    void allReduceMinU64(uint64_t* buf, size_t count, cudaStream_t s);                               // ID-projection keys (GlobalProjection.cpp:66-95)
};
void shardUniqueId(unsigned char* out128);
void launch_pack_rows(const LifeParams& lp, float* table, Enq q);
void launch_lifecycle(const LifeParams& lp, const float* gathered, FrameResult* res, Enq q);
void launch_set_count(uint32_t* c, uint32_t v, Enq q);

class Model {
public:
    // ghost = replica of a model whose surfel store lives on another rank (SURVEY 8e): pose, ids and age only, no device buffers
    Model(MaskFusion* owner, unsigned char id, float confidenceThresh, bool enableFillIn, int capacity, int ownerRank = 0, bool ghost = false);
    Model(const Model&) = delete;

    // ---- reference API (Core/Model/Model.h:128-164) ----
    void initialise(int time);                                        // Model::initialise (+ computeFeedbackBuffers)
    void prepareTracking();                                           // Model::initICP (model side)
    void predictIndices(int time, float depthCutoff, int timeDelta, bool forClean = true);  // Model::predictIndices (forClean: also the packed window texels)
    void fuse(int time, float depthCutoff, float weightMultiplier);   // Model::fuse
    void clean(int time, int timeDelta, float depthCutoff);           // Model::clean
    void combinedPredict(float depthCutoff, int time, int maxTime, int timeDelta);   // Model::combinedPredict + performFillIn
    void overridePose(const Mat4& p) { lastPose = pose; pose = p; pushPose(); }
    void makeStatic(const Mat4& globalPose) { initialC2Winv = mul(pose, rigidInverse(globalPose)); isStatic = true; }
    void updateStaticPose(const Mat4& globalPose) { overridePose(mul(initialC2Winv, globalPose)); }
    void pushPose();                                                  // host pose/lastPose -> device-resident DevPose (k_set_pose)
    bool allowsFillIn() const { return fillIn; }
    unsigned lastCount();                                             // Model::lastCount (synchronises)
    SurfelPlanes planes(int b) const { return SurfelPlanes{pos[b].p, col[b].p, nrm[b].p}; }
    SurfelPlanes current() const { return planes(target); }
    uint32_t* dCount() const { return count.p + countSel; }

    MaskFusion* owner;
    int ownerRank = 0; bool owned = true;                             // sharded mode: which rank holds the surfels
    unsigned char id; int classID = -1;
    Mat4 pose, lastPose, initialC2Winv;
    bool isStatic = false, nonstatic = false; unsigned age = 0;
    float confidenceThreshold, maxDepth;
    bool fillIn;
    uint32_t capacity;
    int target = 0, countSel = 0;
    DevBuf<float4> pos[2], col[2], nrm[2];
    DevBuf<uint32_t> count;                 // [2] ping-pong, device-resident (no host round trip in the loop)
    HostBuf<uint32_t> hCount;               // pinned mirror
    // index map
    DevBuf<uint64_t> key;
    DevBuf<uint32_t> idx; DevBuf<float4> vertConf, colorTime, normRad, cleanTex;
    // prediction + fill-in
    DevBuf<uchar4> splatImage, fillImage; DevBuf<float4> splatVertex, splatNormal, fillVertex, fillNormal; DevBuf<uint16_t> splatTime;
    DevBuf<uint32_t> nonBlack;
    // association
    DevBuf<uint8_t> aflag; DevBuf<uint32_t> abest; DevBuf<float4> meas[3]; DevBuf<uint32_t> slot;
    DevBuf<uint8_t> keep; DevBuf<uint32_t> blockSums, blockSums2, cand, candCount;
    HostBuf<uint32_t> hCleanStat;            // pinned: {first moved sub-block, sub-blocks} of the previous clean (adaptive in-place / copy choice)
    DevBuf<uint32_t> cleanTicket, cleanLoaded; uint32_t cleanEpoch = 0;     // in-place compaction of Model::clean: [0] ticket, [1] first moved sub-block; published epochs
    // tracking
    DevBuf<float4> vmapG[3], nmapG[3], cloud[3];
    DevBuf<float> lastDepth[3]; DevBuf<uint8_t> lastImage[3]; DevBuf<uint8_t> lastNextImage2;
    DevBuf<DataTerm> corres[3];
    DevBuf<uint32_t> validBits[3];           // object models: validity bitmask of nmapG (see k_valid_bits3)
    DevBuf<TrackState> trackState; DevBuf<float> partial;
    DevBuf<DevPose> dpose;                  // what every kernel reads: pose, inverse, fusion weight (device resident)
    HostBuf<float> hTrackOut;               // pinned: pose(16) transform(16) stats(8)
    Mat4 lastTransform;
    std::vector<double> poseLog;            // 8 doubles per entry
    bool tracked = false;                   // took part in the tracking launch of the frame in flight (deferred bookkeeping)
    // predictIndices(forClean) is lazy: when Model::clean follows with the same time gate (the frame schedule, MaskFusion.cpp:550-562) the
    // projection rides inside the clean pass; any reader of the index map in between (fuse, the read-backs) runs it stand-alone first
    bool idxDeferred = false; int idxTime = 0, idxDelta = 0; float idxDepth = 0.f;
    int cleanTexTime = -1; float cleanTexConf = -1.f;    // the time / confidence threshold the packed window texels (cleanTex) were written with
    void flushIndex();
};

class MaskFusion {
public:
    MaskFusion(const mf_config& cfg, int device, cudaStream_t stream);
    ~MaskFusion();

    // bool MaskFusion::processFrame(FrameDataPointer, const Eigen::Matrix4f* inPose, float weightMultiplier, bool bootstrap)
    bool processFrame(const uint8_t* rgb, const float* depth, int64_t timestamp, const uint8_t* mask, const Mat4* inPose,
                      float weightMultiplier, bool bootstrap, bool inputsOnDevice);
    // upload + filterDepth; generateCUDATextures; frame side of initRGB.  `s` = stream to enqueue on (nullptr: the main stream)
    void setFrame(const uint8_t* rgb, const float* depth, const uint8_t* mask, bool onDevice, cudaStream_t s = nullptr);
    void uploadInputs(int slot, const uint8_t* rgb, const float* depth, const uint8_t* mask, int64_t timestamp, bool onDevice, cudaStream_t s = nullptr);
    void preprocess(cudaStream_t s = nullptr);
    void generateCUDATextures(cudaStream_t s = nullptr);                                          // Model::generateCUDATextures
    void frameIntensity(cudaStream_t s = nullptr);                                                // RGBDOdometry::initRGB (frame side) + Sobel + validity
    void trackModels(const std::vector<Model*>& ms, bool viaResult = false);                      // performTracking for a batch
    void predict();                                                                               // MaskFusion::predict
    void sync();
    // The tracked pose reaches the host through an asynchronous copy + event recorded right after the tracking kernel.  The -static
    // schedule has no host decision that depends on it, so processFrame returns with the rest of the frame enqueued and the pose is
    // picked up (finalisePending) by the next processFrame / getPose / sync; the multi-model schedule finalises inside the frame.
    void finalisePending();
    void logPoses(int64_t timestamp);
    bool pendingTrack = false, pendingLog = false; int64_t pendingTimestamp = 0; std::vector<Model*> pendingModels; Event trackDone;
    // ---- multi-model path (MaskFusion.cpp:287-375) ----
    void globalProjection();                                                                      // GlobalProjection::project + downloadDirect (stays on the device)
    void checkModelCount() const;                                                                 // the ID projection and segmentation hold up to 63 models
    SegModels segModels();                                                                        // the model list of this frame (ids, classes, next id)
    void segTables(const SegModels& sm);
    void edgeMaps();                                                                              // MfSegmentation floatEdgeMap -> binary -> close -> invert
    void performSegmentation(const SegModels& sm, bool allowNew);                                 // MfSegmentation::performSegmentation (result -> FrameResult)
    void segmentEdges(const SegModels& sm, bool allowNew, uint8_t* out);                          // its part after the edge map (also mf_debug_segment)
    unsigned char getNextModelID(bool assign);                                                    // MaskFusion::getNextModelID
    void initFirstRGB(Model* m);                                                                  // RGBDOdometry::initFirstRGB of the current frame
    Model* spawnObjectModel();                                                                    // MaskFusion::spawnObjectModel + moveNewModelToList
    void setFrameClasses(const int32_t* ids, int n) { classIDs.assign(ids, ids + n); }            // FrameData::classIDs

    // ---- a frame in three phases; between them sit the exchanges of the object-sharded mode (SURVEY 8e):
    //   frameBegin  inputs (+ frame-packet broadcast), preprocessing, tracking of the models whose store lives here, pose rows
    //   [pose-row all-gather]
    //   frameProject  device-side lifecycle (inactivation, static poses), local part of the global ID projection
    //   [64-bit MIN all-reduce of the projection keys]
    //   [detector frames: broadcast of frameMask | FrameHdr from the detector rank]
    //   frameEnd  resolve, segmentation + vote (device driven), FrameResult copy, fusion of the local stores, prediction
    // With an NCCL communicator (initShardComm) the exchanges are issued from here on the context's stream and NOTHING in a frame
    // waits for the host; without one the caller moves the rows / keys itself between the phase calls (any transport: the gloo tests).
    void configureShard(int rank, int world);
    void initShardComm(const unsigned char* id128, int rank, int world);
    // returns whether the call processed a frame (with a frame queue, the first length - 1 calls only push theirs)
    bool frameBegin(const uint8_t* rgb, const float* depth, int64_t timestamp, const uint8_t* mask, const Mat4* inPose, bool bootstrap, bool onDevice);
    void getShardPoses(float* out);                             // [MF_MAX_MODELS][32] rows of this rank (external transport; synchronises)
    void setShardPoses(const float* gathered);                  // [world][MF_MAX_MODELS][32] -> device (external transport)
    void frameProject();
    void frameEnd(float weightMultiplier);
    // deferred bookkeeping of the multi-model schedule: applied at the start of the next frame (or by any query in between)
    void applyFrameResult();
    LifeParams lifeParams() const;
    ShardComm shard; bool shardNccl = false;
    // Mask R-CNN backbone on the frame path (MaskRCNN::executeSequential, MaskRCNN.cpp:147-151, is called from MfSegmentation.cpp:130):
    // every k-th frame the RGB image is letter-boxed into the backbone's input and the ResNet-101-FPN forward is enqueued on the
    // backbone's own stream, next to the dense pipeline of the same GPU (the reference runs its network as a ~5 Hz sidecar)
    mf_backbone* backbone = nullptr; int backboneEvery = 0;      // borrowed: the caller owns the handle and its stream
    void attachBackbone(mf_backbone* bb, int everyK);
    // Mask R-CNN detector on the frame path (MfSegmentation.cpp:128-131): a segmentation frame that the caller gave no mask runs the
    // detector every k-th tick on the detector's (= its backbone's) stream; k_frame_masks writes the id image and class list into the
    // frame's mask / header in its slot; the main stream waits (the slot's netDone) just before segmentation reads them.
    mf_detector* detector = nullptr; int detectorEvery = 0;      // borrowed: the caller owns the handle and its stream
    void attachDetector(mf_detector* det, int everyK);
    // the backbone and the detector share one network stream and read one RGBA copy of the frame (netRGBA, unpacked on that stream)
    void attachNetwork(const char* who, bool asDetector, mf_detector* det);
    void runNetwork(int slot, bool runBackbone);                // the attached network on the frame in `slot`, behind its upload
    void waitHandoff(cudaStream_t s);                           // `s` waits for a pending detector hand-off (mask + header written)
    void waitNetwork();                                         // the host waits until no network reads or writes a slot any more
    DevBuf<uchar4> netRGBA;
    // object-sharded run with a detector (mf_shard_attach_detector): `detector` is set on rank detRank only, detectorEvery on every rank.
    // A frame exchanges masks (fExchange) when detRank >= 0, the context is multi-model, the frame tracks and tick % detectorEvery == 0:
    // replicated host state, so every rank issues the same collectives.  The detector rank then runs the detector whatever the caller
    // passed (the mask exists on rank 0 only; FrameHdr::maskGiven keeps it on the device) and its frameMask | FrameHdr goes to every rank.
    int detRank = -1; bool fExchange = false, maskCommPending = false;
    void attachShardDetector(mf_detector* det, int everyK, int detectorRank);
    bool shardFrameMasks(void** ptr, size_t* bytes);            // external transport: the range to broadcast from detRank on this frame
    // overlapped frames run the inputs / preprocessing (and, sharded, every collective) on preStream (MaskFusion::processFrame)
    bool spawnedInApply = false, commOnPre = false; Event evMain, evComm;
    void waitMain(cudaStream_t s);                              // `s` waits for the work queued on the main stream so far
    cudaStream_t commStream();                                  // the stream of the next collective, ordered behind the main stream
    void joinComm(bool now);                                    // the main stream waits for it: now, or where segmentation reads the mask
    HostBuf<FrameResult> hRes; DevBuf<FrameResult> dRes; Event resEvt; bool pendingResult = false;
    DevBuf<float> poseTable, gathered;
    float fWeight = 1.f; int fTick = 0; bool fTracked = false;
    std::vector<std::unique_ptr<Model>> inactiveModels;        // MaskFusion::inactiveModels (MaskFusion.cpp:699-713): kept for exportPoses / savePly
    bool enableSmartModelDelete = true; unsigned modelKeepMinSurfels = 4000; float modelKeepConfThreshold = 0.3f;   // MaskFusion.h:398,414-415
    void projectLocal(); void projectResolve();                 // the two halves of globalProjection()
    static int pickOwner(const int64_t* loads, int world);      // least-loaded rank (by owned surfel capacity), ties -> highest rank
    int rank = 0, world = 1;
    int64_t fTimestamp = 0; Mat4 fInPose; bool fHasPose = false, fBootstrap = false;

    mf_config cfg; Cam cam; int W, H, P; int device;
    cudaStream_t stream;                    // the main stream: the caller's (borrowed) or ownedStream
    Stream ownedStream;
    int tick = 1;
    unsigned trackEpoch = 0;                // flag epoch of the tracker's partial-row exchange (launch_tracking), one per launch
    LaunchRecord rec;
    Enq on(cudaStream_t s = nullptr) { return Enq{s ? s : stream, &rec}; }     // where this context's launches go (nullptr: the main stream)
    std::vector<std::unique_ptr<Model>> models;
    unsigned char nextID = 0;
    // frame
    // The loader's data of one frame is ONE contiguous device buffer, a frame packet -- rgb (3P) | raw depth (4P) | instance mask (P) |
    // FrameHdr -- which is exactly what the object-sharded mode broadcasts (MaskFusion.cpp:212-217).  The packets live in a ring of
    // max(queueLength, 1) + 1 slots: the frames queued by -frameQ (MaskFusion::frameQueue, MaskFusion.cpp:206-209) and the frame processed
    // last, which the deferred spawn (applyFrameResult) and the -static schedule's overlapped tail still read.  Without a queue the ring has
    // two slots: in the -static schedule the upload and preprocessing of frame t+1 run on their own stream (preStream) while the surfel
    // passes of frame t, which still read frame t's images, occupy the main stream.  The attached network runs when a frame is pushed and
    // writes its hand-off into the frame's own slot.  The filtered depth and the RGBA copy are derived per processed frame, in two sets.
    struct FrameSlot {
        DevBuf<uint8_t> packet;
        Event uploaded;                     // the packet is written: the processing stream (if another one) and the network wait for it
        Event netDone;                      // the network has read the packet and (detector) written its mask and header
        cudaStream_t upStream = nullptr;    // stream of the upload (borrowed: the main stream or preStream)
        bool netUsed = false;               // netDone has been recorded: a reuse of the slot waits for it
        bool handoff = false;               // a detector writes this frame's mask / header: segmentation waits for netDone
        int64_t timestamp = 0;
        FrameSlot(size_t bytes, cudaStream_t s);
    };
    std::vector<std::unique_ptr<FrameSlot>> ring;
    int curSlot = 0, queued = 0, queueLength = 0;    // slot of the frame being (or last) processed; frames queued after it; -frameQ
    void setFrameQueue(int length);
    void pushFrame(const uint8_t* rgb, const float* depth, int64_t timestamp, const uint8_t* mask, bool onDevice, cudaStream_t s, int ptick, bool detWanted);
    void popFrame(cudaStream_t s);
    Event retired; bool retiredValid = false;   // main stream at the last pop: frames processed before it are done with their data
    DevBuf<uchar4> rgbBuf[2]; DevBuf<float> depthFiltBuf[2];
    uint8_t* rgb3 = nullptr; uchar4* rgb = nullptr; float* depthRaw = nullptr; float* depthFilt = nullptr;   // the current frame
    uint8_t* frameMask = nullptr; FrameHdr* dHdr = nullptr;                                                   // FrameData::mask / classIDs of the current frame
    int curSet = 0;
    size_t packetBytes() const { return (size_t)P * 8 + sizeof(FrameHdr); }
    uint8_t* slotMask(int k) const { return ring[k]->packet.p + (size_t)P * 7; }
    FrameHdr* slotHdr(int k) const { return reinterpret_cast<FrameHdr*>(ring[k]->packet.p + (size_t)P * 8); }
    void selectSlot(int k)
    {
        curSlot = k; rgb3 = ring[k]->packet.p; depthRaw = reinterpret_cast<float*>(rgb3 + (size_t)P * 3); frameMask = slotMask(k); dHdr = slotHdr(k);
    }
    void selectSet(int k) { curSet = k; rgb = rgbBuf[k]; depthFilt = depthFiltBuf[k]; }
    Stream preStream; Event preDone, inputsCopied; bool preWaitPending = false, copyPending = false;
    cudaEvent_t inputReady = nullptr;        // caller's producer event for device inputs (mf_set_input_event, borrowed): waited on before the next frame's copies
    DevBuf<uint8_t> mask;
    DevBuf<float> depthPyr[3]; DevBuf<float4> vmap[3], nmap[3];
    DevBuf<uint8_t> nextImage[3]; DevBuf<short2> nextGrad[3]; DevBuf<uint8_t> rgbValid[3];
    DevBuf<float> edgeMap; DevBuf<uint8_t> edgeBinary, edgeBuf, edgeInv;
    DevBuf<TrackJob> dJobs; HostBuf<TrackJob> hJobs;
    DevBuf<uint8_t> initFlagR, initFlagF;
    DevBuf<float> scratch;                  // read-back staging
    DevBuf<float4> rayTab;                  // viewing ray of every pixel centre (camera constant): read by the splat rasteriser
    bool frameMapsValid = false, intensityValid = false;
    // multi-model state
    std::vector<int32_t> classIDs;          // of the frame being processed
    int spawnOffset = 0;
    DevBuf<uint64_t> projKeys; DevBuf<uint8_t> projectedIDs;
    DevBuf<int> ccL, ccDense, ccLabA, ccLabB, ccArea, ccBox, mapToMask, absorbId, maskPixels, compModel, compMask;
    DevBuf<uint32_t> ccCounter; DevBuf<unsigned> maskOverlap;
    DevBuf<uint8_t> segTmp, ignoreMap, tblIdToIndex, tblIndexToId, tblIsModel, tblMaskToID, tblIsPerson;
    float minMaskModelOverlap = 0.05f; int minMappedComponentSize = 160; int personClassID = 255;   // MfSegmentation.cpp:43, MfSegmentation.h:58
};

}  // namespace mfb
