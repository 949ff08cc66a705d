/*
 * include/maskfusion_b200.h -- C ABI of the H100-native MaskFusion dense pipeline.
 *
 * The reference has no FFI: its hot path sits behind C++ methods of libmaskfusion.so
 * that take Eigen / OpenCV / OpenGL types (SURVEY.md section 8(b)).  This header is
 * the flat, toolchain-neutral boundary a maintainer binds instead; each entry point
 * names the reference method it replaces.  Plain pointers and sizes only: no torch,
 * Eigen, OpenCV or GL types.  All functions return 0 on success, non-zero on error
 * (text via mf_last_error(), which keeps one message per calling thread); no C++
 * exception leaves a function, and nothing calls exit() (the reference does on CUDA
 * errors, Core/Cuda/convenience.cuh:76-83).
 *
 * Conventions
 *   rgb    : H x W x 3 uint8, as FrameData::rgb (CV_8UC3)      Core/FrameData.h:37
 *   depth  : H x W float32 metres, as FrameData::depth (CV_32FC1) Core/FrameData.h:38
 *   mask   : H x W uint8 (optional external segmentation)      Core/FrameData.h:36
 *   poses  : float[16] COLUMN-major == Eigen::Matrix4f storage (Core/Model/Model.h:263-264)
 *   surfels: 12 floats each, position.xyz conf | colour unused initTime lastTime |
 *            normal.xyz radius                                 Core/Model/Model.h:190-192
 *   "tex4" : H x W x 4 float32, the layout of the reference's RGBA32F GL textures
 *   planar maps: 3*H x W float32 (x plane, y plane, z plane)   Core/Cuda/cudafuncs.cu:124-126
 */
#ifndef MASKFUSION_B200_H
#define MASKFUSION_B200_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define MF_ABI_VERSION 1

/* Effective parameters of one run: the reference spreads these over MaskFusion's
 * 23-argument constructor (Core/MaskFusion.h:47-53), ~60 setters and the GUI
 * defaults pushed every frame (GUI/MainController.cpp:528-571, GUI/Tools/GUI.h). */
typedef struct mf_config {
    int32_t width, height;                 /* Resolution::setResolution, MainController.cpp:117 */
    float fx, fy, cx, cy;                  /* Intrinsics::setIntrinics,  MainController.cpp:124-126 */
    float depthCutoff;                     /* GUI.h:194 = 4.0 */
    float maxDepthProcessed;               /* MaskFusion.cpp:57 = 20.0 */
    float icpWeight;                       /* GUI.h:195 = 20.0 (100 => ICP only, RGBDOdometry.cpp:236-237) */
    int32_t rgbOnly, pyramid, fastOdom, so3, frameToFrameRGB;
    float confGlobal, confObject;          /* MainController.cpp:215-216 = 10, 0.01 */
    int32_t timeDelta;                     /* MainController.cpp:399 = INT_MAX/2 (open loop) */
    float outlierCoeff;                    /* GUI.h:196 = 0.1 */
    int32_t capacityGlobal, capacityObject;/* Core/CMakeLists.txt:27-28 (runtime here, not compile time) */
    int32_t enableMultipleModels;          /* 0 == "-static" */
    int32_t trackAllModels;                /* GUI.h:344 */
    int32_t modelSpawnOffset;              /* GUI.h:347 = 22 */
    float minRelSizeNew, maxRelSizeNew;    /* GUI.h:345-346 */
    float segThreshold, segWeightDistance, segWeightConvexity;           /* GUI.h:367-374 */
    int32_t segMorphEdgeIterations, segMorphEdgeRadius, segMorphMaskIterations, segMorphMaskRadius;
} mf_config;

typedef struct mf_context mf_context;

const char* mf_last_error(void);
int mf_abi_version(void);
void mf_config_defaults(mf_config* cfg, int width, int height);

/* MaskFusion::MaskFusion (Core/MaskFusion.h:47-53).  device = CUDA ordinal
 * (reference: MASKFUSION_GPU_SLAM, MaskFusion.cpp:89-90); stream = cudaStream_t the
 * whole pipeline is enqueued on (NULL = a private non-blocking stream). */
mf_context* mf_create(const mf_config* cfg, int device, void* stream);
void mf_destroy(mf_context* ctx);

/* bool MaskFusion::processFrame(FrameDataPointer, const Eigen::Matrix4f* inPose,
 *      float weightMultiplier, bool bootstrap)                 Core/MaskFusion.h:69-70
 * Host buffers; the H2D copies are part of the call. mask / in_pose may be NULL. */
int mf_process_frame(mf_context* ctx, const uint8_t* rgb, const float* depth, int64_t timestamp,
                     const uint8_t* mask, const float* in_pose, float weight_multiplier, int bootstrap);
/* Same, inputs already resident in device memory (rgb: packed 3 bytes/pixel).
 * Lifetime / ordering of device inputs: the library copies them into its own frame set at the START of the call; on -static
 * tracking frames that copy runs on a private pre-processing stream next to the previous frame's surfel passes, NOT behind
 * the work queued on the context stream.  Therefore (a) the buffers must be completely written when the call is made -- or
 * the producer's completion event is handed over with mf_set_input_event before the call; (b) work the caller enqueues on
 * the CONTEXT stream after the call returns is ordered after the copies (the context stream waits for them), so the buffers
 * may be overwritten from there; a caller writing them from another stream waits for mf_sync or the next call's return. */
int mf_process_frame_device(mf_context* ctx, const void* d_rgb, const void* d_depth, int64_t timestamp,
                            const void* d_mask, const float* in_pose, float weight_multiplier, int bootstrap);
/* cudaEvent_t that the NEXT mf_process_frame_device waits on (on whichever stream it copies from) before it reads its
 * device inputs; consumed by that call.  NULL clears it. */
int mf_set_input_event(mf_context* ctx, void* cuda_event);
int mf_sync(mf_context* ctx);                       /* wait for everything enqueued so far */
int mf_tick(mf_context* ctx);                       /* MaskFusion::getTick */
/* Frame queue, the reference's queueLength (-frameQ, default 30 there; MaskFusion.cpp:37,200-209, MainController.cpp:223,242).  Every
 * mf_process_frame[_device] call pushes its frame; while fewer than `length` frames are queued the call returns without processing
 * anything (mf_tick, poses and the pose log do not change); otherwise it processes the oldest queued frame.  The frame processed by the
 * n-th call of a run is the frame of call n - length + 1, at tick n - length + 1.  length 0 or 1: no queue (the default).
 *   - With the frame travel rgb, depth, the caller's mask, the class list set by mf_set_frame_classes before the call, and the
 *     timestamp.  Host inputs are free when the call returns; device inputs are copied at push time (mf_set_input_event applies).
 *   - in_pose, weight_multiplier and bootstrap belong to the CALL and apply to the frame it processes, not to the frame it pushes (as
 *     in the reference, whose processFrame takes them next to the FrameData it queues).
 *   - An attached detector or backbone runs when the frame is pushed, on the tick the frame will be processed at, and writes its masks
 *     into the queued frame: with a queue its work overlaps the processing of the frames ahead of it.
 *   - Frames still queued at mf_destroy are dropped (the reference never processes the last length - 1 frames of a run).
 *   - Allowed before the first processed frame, with nothing queued; the memory is (max(length, 1) + 1) * (8 * width * height + 1048)
 *     bytes and is allocated here.  Refused: a negative length, and a sharded context (mf_shard_configure with world > 1 or
 *     mf_shard_comm_init), which in turn refuse a context with a queue.  While frames are queued, mf_set_frame and the stage-wise
 *     mf_model_* calls are refused. */
int mf_set_frame_queue(mf_context* ctx, int length);
int mf_frame_queue_size(mf_context* ctx);           /* frames queued and not yet processed: whether a call processed a frame */
int64_t mf_kernel_launches(mf_context* ctx);        /* kernels launched since creation */

/* ---- model list (MaskFusion::getModels) ---- */
int mf_model_count(mf_context* ctx);
int mf_model_id(mf_context* ctx, int i);
int mf_get_pose(mf_context* ctx, int i, float pose16[16]);          /* Model::getPose */
int mf_set_pose(mf_context* ctx, int i, const float pose16[16]);    /* Model::overridePose */
int mf_model_surfel_count(mf_context* ctx, int i);                  /* Model::lastCount */
int mf_model_set_conf_threshold(mf_context* ctx, int i, float t);   /* Model::setConfidenceThreshold */
int mf_download_surfels(mf_context* ctx, int i, float* out, int max_surfels);   /* Model::downloadMap, Model.cpp:944-974 */
int mf_upload_surfels(mf_context* ctx, int i, const float* in, int n);          /* test / bootstrap hook */
int mf_pose_log_size(mf_context* ctx, int i);                                   /* Model::getPoseLog */
int mf_get_pose_log(mf_context* ctx, int i, double* out8, int max_entries);     /* ts x y z qx qy qz qw, MaskFusion.cpp:850-879 */

/* ---- per-stage entry points (same names / order as Core/Model/Model.h:128-164) ---- */
int mf_set_frame(mf_context* ctx, const uint8_t* rgb, const float* depth, const uint8_t* mask);   /* upload + filterDepth + Model::generateCUDATextures */
int mf_model_perform_tracking(mf_context* ctx, int i, float transform16[16]);                      /* Model::performTracking */
int mf_model_predict_indices(mf_context* ctx, int i, int time);                                    /* Model::predictIndices */
int mf_model_fuse(mf_context* ctx, int i, int time, float depth_cutoff, float weight_multiplier);  /* Model::fuse */
int mf_model_clean(mf_context* ctx, int i, int time);                                              /* Model::clean */
int mf_model_combined_predict(mf_context* ctx, int i, int time, int max_time);                     /* Model::combinedPredict + performFillIn */
int mf_model_init_from_frame(mf_context* ctx, int i, int time);                                    /* computeFeedbackBuffers + Model::initialise */

/* ---- read-back of intermediate products, in the reference's layouts ---- */
int mf_download_filtered_depth(mf_context* ctx, float* out);                                       /* textureDepthMetricFiltered */
int mf_download_frame_maps(mf_context* ctx, int level, float* depth, float* vmap_planar, float* nmap_planar);  /* GPUSetup::{depth,vertex_map,normal_map}_tmp */
int mf_download_model_maps(mf_context* ctx, int i, int level, float* vmap_planar, float* nmap_planar);          /* RGBDOdometry::vmaps_g_prev_/nmaps_g_prev_ */
int mf_download_index_map(mf_context* ctx, int i, uint32_t* idx, float* vert_conf4, float* color_time4, float* norm_rad4); /* ModelProjection sparse* textures */
int mf_download_prediction(mf_context* ctx, int i, uint8_t* image4, float* vertex_conf4, float* normal_rad4, uint16_t* time); /* splat textures */
int mf_download_fill_in(mf_context* ctx, int i, uint8_t* image4, float* vertex4, float* normal4);  /* FillIn textures */
int mf_download_association(mf_context* ctx, int i, uint8_t* update_id, uint32_t* best, float* meas12); /* x-major pixel order, Model.cpp:179-183 */
int mf_download_track_stats(mf_context* ctx, int i, double* A36, double* b6, float* err_count6);   /* RGBDOdometry::lastA/lastb, lastICPError,... */
int mf_download_edge_map(mf_context* ctx, float* edge, uint8_t* binary);                           /* MfSegmentation floatEdgeMap / binary edge map */
/* test hook: morphological close of a host image (W x H of the context, in place). ellipse != 0: cv::morphologyEx(MORPH_CLOSE, MORPH_ELLIPSE) of the
 * mask-id image (MfSegmentation.cpp:424-426); ellipse == 0: the binary edge-map close (segmentation.cu:217-255,334-354), `inverted` = 255 - result. */
/* Mask R-CNN backbone on the frame path (MaskRCNN::executeSequential, MaskRCNN.cpp:147-151, called at MfSegmentation.cpp:130): every k-th
 * processFrame letter-boxes the frame's RGB image into `backbone`'s input (mf_backbone_mold) and enqueues its forward on the backbone's
 * own stream, concurrently with the dense pipeline on the same GPU.  backbone = handle of mf_backbone_create; NULL detaches.
 * Refused: a -static context (it runs no segmentation to feed), and a context with a detector attached. */
int mf_attach_backbone(mf_context* ctx, void* backbone, int every_k);
/* Mask R-CNN detector on the frame path: MfSegmentation::performSegmentation calls MaskRCNN::executeSequential when the frame has no mask
 * (MfSegmentation.cpp:128-131), which fills FrameData::mask with the id image and FrameData::classIDs with [0] followed by the exported class
 * ids (MaskRCNN.cpp:98-151).  With a detector attached (handle of mf_detector_create), a frame runs it when the context is multi-model,
 * the caller passed NO mask, the frame runs segmentation (tick > 1 and not an in_pose frame) and mf_tick() % every_k == 0 before the call
 * (with a frame queue: the tick the frame is processed at; whether the processing call passes an in_pose is not known yet, and such a
 * frame's detection goes unused).  Detection (mould, backbone, RPN, heads at the context's W x H) and the hand-off into the frame's mask and
 * class list are enqueued on the detector's stream behind the frame's upload; the context's stream waits for them only where segmentation first reads the mask,
 * so tracking and the ID projection overlap the detector.  Nothing in the frame waits for the host.
 *   - A frame skipped by every_k carries no masks (as with mask = NULL and no detector).  A frame given a mask uses it and the classes of
 *     mf_set_frame_classes; the detector does not run.
 *   - A failing export rule (special_assignments[class_id] out of range, an IndexError upstream) leaves that frame without masks, and the
 *     NEXT call on the context returns non-zero with the message.
 *   - Refused: a -static context, world > 1 (sharded runs use mf_shard_attach_detector), a backbone attached (and mf_attach_backbone while
 *     a detector is attached); mf_shard_configure and mf_shard_comm_init refuse a context with a detector attached here.
 *   - NULL detaches; detaching and mf_destroy first wait for the last hand-off.  The context never destroys the detector: detach (or destroy
 *     the context) before destroying it.  Detector launches (the frame's RGBA copy it reads included) are not counted in mf_kernel_launches. */
struct mf_detector;
int mf_attach_detector(mf_context* ctx, struct mf_detector* detector, int every_k);
/* FrameData::mask (W x H) and classIDs (n_masks entries of class_ids_256) that segmentation read on the last frame; mask is all zero when
 * n_masks is 0 (the frame carried no masks).  NULL skips an output.  Multi-model contexts only. */
int mf_download_frame_masks(mf_context* ctx, uint8_t* mask, int32_t* class_ids_256, int* n_masks);
int mf_debug_track_timing(int64_t* out, int cap);   /* profiling builds only (-DMF_TRACK_TIMING): (tag, SM clock) pairs of the last tracking launch; else 0 */
int mf_morph_close(mf_context* ctx, uint8_t* image, int radius, int iterations, int ellipse, uint8_t* inverted);

/* ---- stand-alone kernels exposed for parity tests (device work, host buffers) ---- */
/* ---- multi-model inputs / outputs ---- */
int mf_set_frame_classes(mf_context* ctx, const int32_t* class_ids, int n);   /* FrameData::classIDs of the NEXT processFrame call (classIDs[mask value]; entry 0 = background), Core/FrameData.h:40 */
int mf_download_segmentation(mf_context* ctx, uint8_t* mask, uint8_t* projected_ids);   /* SegmentationResult::fullSegmentation (textureMask) and GlobalProjection::getProjectedModelIDs */
int mf_model_class_id(mf_context* ctx, int i);                                /* Model::getClassID */

/* ---- object-sharded mode: one context per GPU/rank, object Models (and their surfel stores) partitioned over the ranks
 *      (BASELINE.json north_star "Object Models ... shard one-per-GPU"); the couplings of a frame are exactly those of
 *      MaskFusion.cpp:212-217 (every model reads the frame), :257-276 (tracked poses decide inactivation; static objects follow the
 *      global pose), GlobalProjection.cpp:66-95 (one depth-tested ID image) and MaskFusion.cpp:296-297 (one segmentation, evaluated
 *      identically on every rank from the merged image).
 *
 *      (1) In-library exchange (the product path): after mf_shard_comm_init every rank calls mf_shard_process_frame once per frame;
 *          only rank 0 passes inputs.  The library issues, on the context's stream and without any host synchronisation inside the
 *          frame: ncclBroadcast of the frame packet (rgb | depth | mask | header, one buffer), ncclAllGather of the pose rows of the
 *          tracked models, ncclAllReduce(ncclMin, ncclUint64) of the ID-projection keys.  libnccl.so.2 is opened at run time.
 *          Bootstrap: rank 0 calls mf_shard_unique_id and distributes the 128 bytes by any side channel (the tests and bench.py use
 *          torch.distributed's store); the communicator lives in the context.
 *      (2) Transport-agnostic phases (tests over gloo, one GPU or none of the NCCL requirements): the caller moves the data itself
 *              [frame to every rank]  mf_set_frame_classes; mf_shard_frame_begin;
 *              mf_shard_get_poses -> [all-gather of 64 x 32 floats] -> mf_shard_set_poses;
 *              mf_shard_project -> [MIN all-reduce of the uint64 keys at mf_shard_projection_keys];
 *              mf_shard_frame_masks -> [if it returns 1: broadcast of the returned device range from the detector rank];
 *              mf_shard_frame_end
 *      With world == 1 the three phase calls are exactly mf_process_frame.
 *
 *      Detector (mf_shard_attach_detector): the Mask R-CNN runs on one rank, detector_rank.  A frame exchanges masks when the context
 *      is multi-model, the frame tracks (tick > 1) and mf_tick() % every_k == 0 -- every rank evaluates this on replicated state.  On such
 *      a frame the detector rank detects and hands off into its copy of the frame (a caller's mask, sent with the packet, takes
 *      precedence on the device: the network still runs, its output is dropped), and a fourth exchange broadcasts that rank's
 *      mask | header (width*height + header bytes) to every rank: in (1) an ncclBroadcast on the context's stream after the key
 *      all-reduce, in (2) the range mf_shard_frame_masks returns.  Every rank then computes what one process with mf_attach_detector
 *      and the same every_k computes, bit for bit; an export error of the detector surfaces on every rank on the next call.  New object
 *      models prefer ranks other than the detector rank (it counts one more tracked model in the placement rule). ---- */
int mf_shard_configure(mf_context* ctx, int rank, int world);                 /* before the first frame; rank 0 owns the background model */
int mf_shard_unique_id(uint8_t* out128);                                      /* ncclGetUniqueId (rank 0) */
/* ncclCommInitRank on the context's device (+ mf_shard_configure).  Refused, whatever the world size: a -static context (one model, nothing
 * to shard: run replicas), and a context with a detector attached by mf_attach_detector. */
int mf_shard_comm_init(mf_context* ctx, const uint8_t* id128, int rank, int world);
int mf_shard_process_frame(mf_context* ctx, const uint8_t* rgb, const float* depth, int64_t timestamp, const uint8_t* mask,
                           const int32_t* class_ids, int n_class_ids, float weight_multiplier,
                           int inputs_on_device);   /* inputs are read on rank 0 only (class_ids always from the host) */
int mf_shard_stats(mf_context* ctx, int64_t* out4);                           /* collective bytes moved, NCCL calls, communicator size, NCCL version */
int mf_shard_frame_begin(mf_context* ctx, const void* rgb, const void* depth, int64_t timestamp, const void* mask, int on_device);
int mf_shard_get_poses(mf_context* ctx, float* out_64x32, int capacity_models);   /* returns nModels; row i = pose(16) lastTransform(16) of model i if it is tracked here, else 0 */
int mf_shard_set_poses(mf_context* ctx, const float* gathered_world_x_64_x32);
int mf_shard_project(mf_context* ctx);                                        /* device-side lifecycle after tracking + local models into the key image */
void* mf_shard_projection_keys(mf_context* ctx);                              /* device pointer, width*height uint64 (depth bits << 32 | model index << 26 | surfel) */
int mf_shard_frame_end(mf_context* ctx, float weight_multiplier);
/* every rank, between the same frames, with the same every_k and detector_rank; detector non-NULL exactly on detector_rank (where
 * detector_reserve_image sizes its id image now).  Needs a sharded multi-model context (world > 1: mf_shard_configure or
 * mf_shard_comm_init first) and no backbone.  (NULL, 0, -1) detaches on every rank; the detector rank first waits for the last hand-off. */
int mf_shard_attach_detector(mf_context* ctx, struct mf_detector* detector, int every_k, int detector_rank);
/* phase call of (2), between mf_shard_project and mf_shard_frame_end: 1 and the device range (frame mask | header) to broadcast from the
 * detector rank when this frame exchanges masks (on the detector rank, the context's stream first waits for the hand-off), else 0.
 * Always 0 with a communicator: the library broadcasts the range itself. */
int mf_shard_frame_masks(mf_context* ctx, void** d_ptr, size_t* bytes);
int mf_model_owner(mf_context* ctx, int i);                                   /* rank holding model i's surfels */
/* CTAs of the persistent tracking launch per tracked model (host only): bit j of light_mask marks an object model (validity bitmask, nearly all
 * pixels culled), the others are full-frame models and get `ratio` times the share.  Model::performTracking of a batch of models (Model.cpp:427-447)
 * is ONE launch here; this is how its grid is dealt.  n_jobs <= 32. */
int mf_track_shares(int n_jobs, unsigned light_mask, int total_ctas, int ratio, int* shares);
int mf_shard_pick_owner(const int64_t* loads, int world);                     /* placement rule for a new model: least owned capacity, ties -> highest rank (host only) */

/* in-stream CUDA-event stage timer (replaces the reference's TICK/TOCK Stopwatch, Core/Utils/Stopwatch.h:46-54) */
int mf_set_profiling(mf_context* ctx, int on);
int mf_get_stage_times(mf_context* ctx, char* buf, int bufsize);   /* lines: "name count total_ms" */
int mf_debug_set_poses(mf_context* ctx, int i, const float pose16[16], const float last_pose16[16]);   /* sets Model::pose and Model::lastPose verbatim */
int mf_icp_step(mf_context* ctx, int i, int level, const float Rcurr9[9], const float tcurr3[3], float out29[29]);  /* icpStep, reduce.cu:446-525 */

/* ---- Mask R-CNN backbone: ResNet-101 + FPN as wgmma GEMMs (replaces the dense part of the Keras/TF sidecar,
 *      Core/Segmentation/MaskRCNN/MaskRCNN.py.in:55-58,101-111; weights are synthetic/seeded unless loaded with mf_*_load_weights).
 *      The Mask R-CNN functions (mf_backbone_*, mf_rpn_*, mf_detector_*, mf_roi_align_bf16) report a refusal or a CUDA failure by returning
 *      -1, a creator by returning NULL, and mf_gemm_bf16 and mf_conv3x3_bf16 by returning -2; mf_last_error() has the text. ---- */
typedef struct mf_backbone mf_backbone;
const char* mf_cnn_last_error(void);      /* the same text as mf_last_error(), under the name kept for existing bindings */
/* Pretrained weights (the reference's model.load_weights(COCO_MODEL_PATH, by_name=True)): a safetensors file of matterport's Keras
 * arrays named "<layer>/<param>", F32, Keras layouts (scripts/convert_mrcnn_h5.py writes it from mask_rcnn_coco.h5; DESIGN §3c has the
 * name table).  BatchNorm is folded on the host (R-FOLD).  Each loader reads its own handle's tensors and ignores the others; all or
 * nothing: everything is read, checked and folded before the handle changes, and on an error (mf_last_error() names the file and the
 * tensor) its weights stay as they were.  The copy is ordered on the handle's stream after the work queued there, and complete on
 * return: safe between frames with the detector attached; mf_*_get_weights read the new tables afterwards.  mf_rpn_load_weights and
 * mf_detector_load_weights are declared with their handles below. */
int mf_backbone_load_weights(mf_backbone* h, const char* path);
/* one handle layer exactly as the loaders fold it, on the host (no CUDA device needed): w [rows x K] (K order (ky, kx, cin), zero padded),
 * bias [rows]; dims = {rows, K}.  Layer names: the Keras conv layer ("conv1", "res4b_branch2a", "fpn_c3p3", "fpn_p2", "rpn_conv_shared",
 * "mrcnn_class_conv1", "mrcnn_mask_conv2", "mrcnn_mask_deconv", "mrcnn_mask", ...) or the stacked pairs "rpn_class_raw+rpn_bbox_pred"
 * and "mrcnn_class_logits+mrcnn_bbox_fc".  w or bias NULL: only dims, the file is not read. */
int mf_mrcnn_read_layer(const char* path, const char* layer, float* w_rows_K, float* bias_rows, int* dims);
/* out[MxN] = relu?(A[MxK] * B[NxK]^T + bias[N] + residual[MxN]); bf16 device pointers, K % 64 == 0, N % 64 == 0 */
int mf_gemm_bf16(const void* dA, const void* dB, const float* dBias, const void* dResidual, void* dOut, int M, int N, int K, int relu, void* stream);
/* implicit-GEMM 3x3/s1/p1 convolution, NHWC bf16, weights [Cout][3][3][Cin]; the activation is read through a 3-D TMA map (no im2col) in
 * boxes of Wbox x Hbox = 128 pixels, Wbox = min(W, 128).  Admitted: Cin a positive multiple of 64, Cout a positive multiple of 64, H > 0, and
 * either W in {8, 16, 32, 64} with H % (128 / W) == 0 or W a multiple of 128 (at most 131072); H * W and 9 * Cin within int.  Any other
 * shape returns -2 without touching the device; the message of an H, W or Cin outside this is "conv3x3: unsupported geometry". */
int mf_conv3x3_bf16(const void* dIn, const void* dW, const float* dBias, const void* dResidual, void* dOut, int H, int W, int Cin, int Cout, int relu, void* stream);
mf_backbone* mf_backbone_create(int input_size, unsigned seed, void* stream);
void mf_backbone_destroy(mf_backbone* h);
int mf_backbone_num_layers(mf_backbone* h);
int mf_backbone_layer(mf_backbone* h, int i, int* cin_cout_k_stride_pad_kpad);
int mf_backbone_get_weights(mf_backbone* h, int i, float* w_cout_kpad, float* bias);
int mf_backbone_mold(mf_backbone* h, const void* d_rgba, int W, int H);            /* letter-box + mean subtraction -> network input */
void* mf_backbone_stream(mf_backbone* h);   /* the cudaStream_t the backbone enqueues on */
void* mf_backbone_input_buffer(mf_backbone* h);
int mf_backbone_forward(mf_backbone* h, const void* d_input_nhwc_bf16);
void* mf_backbone_output(mf_backbone* h, int level, int* dims_hwc);               /* 0..3 = C2..C5, 4..8 = P2..P6 (device, NHWC bf16) */
int mf_backbone_download(mf_backbone* h, int level, void* host_bf16);
double mf_backbone_flops(mf_backbone* h);
int mf_backbone_num_gemms(mf_backbone* h);

/* ---- Mask R-CNN region proposals on the backbone's P2..P6 (matterport mrcnn rpn_graph + ProposalLayer + PyramidROIAlign, COCO
 *      InferenceConfig; weights synthetic/seeded unless loaded, owned by the handle, not by the backbone's layer table).  The handle reads the
 *      backbone's outputs and enqueues on the backbone's stream; destroy it before the backbone.  Errors: mf_last_error().
 *      Anchors: 3 per feature pixel (ratios 0.5, 1, 2), order (level P2..P6, y, x, ratio), normalised y1 x1 y2 x2; A anchors in all.
 *      Boxes are normalised y1 x1 y2 x2 float; pooled features are [n][pool][pool][256] bf16. ---- */
typedef struct mf_rpn mf_rpn;
#define MF_RPN_CONV 1          /* shared 3x3 256->512 conv + ReLU on P2..P6 (wgmma GEMM) */
#define MF_RPN_HEADS 2         /* 1x1 class-logit and box-delta heads as one GEMM with fp32 output -> logits [A][2], deltas [A][4] */
#define MF_RPN_PROPOSALS 4     /* top 6000 by score, decode + clip, NMS 0.7 -> 1000 proposals (zero padded) and the kept count */
#define MF_RPN_ROI_ALIGN 8     /* 7x7 ROI Align of the 1000 proposals */
mf_rpn* mf_rpn_create(mf_backbone* bb, unsigned seed);
int mf_rpn_load_weights(mf_rpn* h, const char* path);          /* rpn_conv_shared, rpn_class_raw, rpn_bbox_pred (see mf_backbone_load_weights) */
void mf_rpn_destroy(mf_rpn* h);
int mf_rpn_forward(mf_rpn* h);                        /* all four stages, after mf_backbone_forward on the same stream */
int mf_rpn_run(mf_rpn* h, int stages);                /* a subset of the stages (MF_RPN_* bits), in order */
int mf_rpn_num_anchors(mf_rpn* h);
/* the proposal stage of the forward on caller-supplied device arrays: logits [n][2], deltas [n][4], anchors [n][4] float, 1 <= n <= A */
int mf_rpn_propose(mf_rpn* h, const float* d_logits, const float* d_deltas, const float* d_anchors, int n_anchors);
/* pyramid ROI Align of n boxes (device, [n][4]) on bb's P2..P5 into d_out ([n][pool][pool][256] bf16, device), 2 <= pool <= 64; bb's stream */
int mf_roi_align_bf16(mf_backbone* bb, const float* d_boxes, int n, int pool, void* d_out);
/* read-back to host memory (each waits for the handle's stream); NULL skips an output */
int mf_rpn_get_weights(mf_rpn* h, float* conv_w_512x2304, float* conv_b_512, float* head_w_18x512, float* head_b_18);   /* (ky,kx,cin) order; head rows 0..5 logits, 6..17 deltas */
int mf_rpn_get_anchors(mf_rpn* h, float* anchors_Ax4);
int mf_rpn_get_head_outputs(mf_rpn* h, float* logits_Ax2, float* deltas_Ax4);
int mf_rpn_download_conv(mf_rpn* h, int level, void* host_bf16);                 /* level 0..4 = P2..P6: H x W x 512 bf16 */
int mf_rpn_get_proposals(mf_rpn* h, float* rois_1000x4);                          /* returns the kept count */
int mf_rpn_get_pooled(mf_rpn* h, void* host_bf16_1000x7x7x256);

/* ---- Mask R-CNN detection heads on an mf_rpn's proposals (matterport mrcnn fpn_classifier_graph + DetectionLayer + build_fpn_mask_graph +
 *      unmold_detections + generate_id_image, COCO InferenceConfig: 81 classes; weights synthetic/seeded unless loaded, owned by the handle).  The handle
 *      reads the RPN's proposals and pooled features and the backbone's P2..P5, and enqueues on the backbone's stream; destroy it before the
 *      RPN.  Errors: mf_last_error().  Shapes are the upstream ones: 1000 ROIs, 100 detection rows.  Detections are [100][6] float
 *      y1 x1 y2 x2 (normalised to the S x S network input, clipped to the letter-box window of the image) class score, zero rows after the
 *      count; masks are [100][28][28] float (sigmoid of the detection's own class).  The image size (W x H, the letter-box window) is the one
 *      given to the last mf_detector_forward / detect / paste; S x S after create. ---- */
typedef struct mf_detector mf_detector;
#define MF_DET_CLASSIFIER 1    /* FC1 (7x7 conv on the pooled ROIs), FC2, class logits + box deltas (one GEMM, fp32) */
#define MF_DET_DETECTIONS 2    /* softmax, refinement, clip to the window, confidence 0.7, per-class NMS 0.3, top 100 -> detections + count */
#define MF_DET_MASKS 4         /* 14x14 ROI Align of the detections, 4 x 3x3 conv, 2x2/s2 transposed conv, 1x1 logits, own-class sigmoid */
#define MF_DET_ID_IMAGE 8      /* unmould to image pixels + generate_id_image (export rule of mf_detector_set_export) -> id image, ids, rois */
mf_detector* mf_detector_create(mf_rpn* rpn, unsigned seed);
int mf_detector_load_weights(mf_detector* h, const char* path);  /* mrcnn_class_*, mrcnn_bbox_fc, mrcnn_mask* (see mf_backbone_load_weights) */
void mf_detector_destroy(mf_detector* h);
int mf_detector_run(mf_detector* h, int stages);                  /* a subset of the stages (MF_DET_* bits), in order */
int mf_detector_forward(mf_detector* h, int image_w, int image_h); /* all stages after mf_rpn_forward, for an image of image_w x image_h */
/* what MaskRCNN.execute() does: mould the W x H RGBA8 device image, backbone, RPN and all head stages, enqueued on one stream */
int mf_detector_detect(mf_detector* h, const void* d_rgba, int W, int H);
/* generate_id_image's min_score, class_filter and special_assignments (mf_generate_id_image's conventions, <= 128 entries each; NULL with
 * count 0 for none).  Default: 0.55 and no lists. */
int mf_detector_set_export(mf_detector* h, double min_score, const int32_t* class_filter, int n_filter, const int32_t* special_assignments,
                           int n_special);
/* the detection layer on caller-supplied device arrays: rois [n][4], logits [n][81], deltas [n][81][4] float, 1 <= n <= 1000; the window
 * of the current image size */
int mf_detector_refine(mf_detector* h, const float* d_rois, const float* d_logits, const float* d_deltas, int n);
/* unmould + id image on caller-supplied device arrays: detections [100][6], masks [100][28][28] float, for a W x H image */
int mf_detector_paste(mf_detector* h, const float* d_detections, const float* d_masks, int W, int H);
/* read-back to host memory (each waits for the handle's stream); NULL skips an output */
int mf_detector_num_layers(mf_detector* h);
/* layer i: Cin, rows (GEMM N, zero rows included), k, stride, pad, K.  0 FC1, 1 FC2, 2 heads (rows 0..80 logits, 81 + 4c + k deltas of class
 * c), 3..6 mask convs, 7 transposed conv (row (dy*2 + dx)*256 + cout), 8 mask logits */
int mf_detector_layer(mf_detector* h, int i, int* cin_rows_k_stride_pad_K);
int mf_detector_get_weights(mf_detector* h, int i, float* w_rows_K, float* bias_rows);   /* (ky,kx,cin) order along K */
int mf_detector_get_fc(mf_detector* h, void* fc1_bf16_1000x1024, void* fc2_bf16_1000x1024);
int mf_detector_get_head_outputs(mf_detector* h, float* logits_1000x81, float* deltas_1000x81x4);
/* mask head layer i: 0 pooled 100x14x14x256, 1..4 conv outputs 100x14x14x256, 5 transposed conv 100x14x14x2x2x256 (bf16); 6 mask logits
 * 100x14x14x2x2x81 (float) */
int mf_detector_get_mask_layer(mf_detector* h, int i, void* host);
int mf_detector_get_detections(mf_detector* h, float* detections_100x6);            /* returns the detection count */
int mf_detector_get_masks(mf_detector* h, float* masks_100x28x28);
/* the execute() outputs in mf_generate_id_image's layout: id image H x W uint8, exported class ids, rois y1 x1 y2 x2 int32 (each sized for
 * 100); returns the exported count */
int mf_detector_get_id_image(mf_detector* h, uint8_t* id_image, int32_t* class_ids, int32_t* rois);
int mf_detector_image_size(mf_detector* h, int* w, int* hgt);

/* ---- image-directory loader ("-dir", GUI/Tools/ImageLogReader.{h,cpp}; GUI/MainController.cpp:150-176) ----
 * colour .png/.ppm/.jpg, depth 16-bit .png (x 0.001), masks 8-bit .png/.pgm + "<mask>.txt" (class ids, boxes); .exr depth is refused
 * (no OpenEXR in this build).  hasMore() lets the last frame through (ImageLogReader.cpp:326), unlike the .klg reader. */
typedef struct mf_dir mf_dir;
mf_dir* mf_dir_open(const char* color_dir, const char* depth_dir, const char* mask_dir /* NULL: no masks */, int index_width /* <=0: 4 */,
                    const char* color_prefix, const char* depth_prefix, const char* mask_prefix);   /* ImageLogReader::ImageLogReader */
int mf_dir_num_frames(mf_dir* r);                                       /* ImageLogReader::getNumFrames */
int mf_dir_has_more(mf_dir* r);                                         /* ImageLogReader::hasMore */
int mf_dir_has_masks(mf_dir* r);                                        /* LogReader::hasMasks */
int mf_dir_set_max_masks(mf_dir* r, int n);                             /* ImageLogReader::setMaxMasks ("-nm") */
int mf_dir_size(mf_dir* r, int* width, int* height);                    /* size of the first colour image */
/* ImageLogReader::getNext + loadFrameFromDrive: rgb HxWx3, depth HxW metres; mask/class_ids/boxes may be NULL.  *n_class_ids: in =
 * capacity, out = ids read (classIDs[0] == 0, ImageLogReader.cpp:306); boxes = cv::Rect x,y,w,h per object.  Returns 1 if a mask was
 * delivered, 0 if not, < 0 on error; timestamp = index * 1000 / 24 (ImageLogReader.cpp:283). */
int mf_dir_get_next(mf_dir* r, uint8_t* rgb, float* depth, uint8_t* mask, int32_t* class_ids, int32_t* boxes, int* n_class_ids, int64_t* timestamp);
void mf_dir_close(mf_dir* r);

/* MaskFusion::exportPoses (Core/MaskFusion.cpp:849-881): writes <export_dir>poses-<model id>.txt for every active model
 * and for every inactivated model the reference's keep rule retained (inactivateModel, MaskFusion.cpp:699-713: smart delete keeps a model
 * with >= 4000 surfels and confidence threshold > 0.3) ("seconds x y z qx qy qz qw", fixed notation, 6 decimals); returns the number of files. */
int mf_export_poses(mf_context* ctx, const char* export_dir);

/* PLY export of one model's surfels as MaskFusion::savePly writes it (Core/MaskFusion.cpp:733-848): vertices with conf > threshold,
 * binary little endian, x y z | r g b | -nx -ny -nz | radius.  surfels = n x 12 floats as mf_download_surfels returns them. */
int mf_write_ply(const char* path, const float* surfels, int n, float conf_threshold);

/* PreSegmentation::performSegmentation (Core/Segmentation/PreSegmentation.cpp:28-90, the "precomputed masks" performer; host code in the
 * reference too): mask values -> model ids through the persistent table `mapping` (256 bytes, zero-initialised by the caller before the first
 * frame; the reference's function-static vector), the first unseen value in raster order becomes next_model_id when allow_new.  Outputs: the full
 * segmentation (W*H), has_new_label, and per model in list order (the new one last) superPixelCount, depthMean, depthStd (mean absolute deviation),
 * the inputs of Model::setMaxDepth (MaskFusion.cpp:291,337-341).  model_ids: ids of the live models, background first.  Returns the number of
 * entries written.  Not wired into the device-driven schedule (its statistics are sequential float sums in raster order). */
int mf_pre_segmentation(const uint8_t* mask, const float* depth, int W, int H, const uint8_t* model_ids, int n_models, int next_model_id,
                        int allow_new, uint8_t* mapping, uint8_t* full_segmentation, int* has_new_label, uint32_t* super_pixel_count,
                        float* depth_mean, float* depth_std);

/* Mask R-CNN post-processing (Core/Segmentation/MaskRCNN/helpers.py:70-98 generate_id_image): detections (masks HxWxN u8, N fastest;
 * scores; class ids; rois N x 4) -> id image HxW (ids 1..n in export order, later detections overwrite earlier ones), exported class ids
 * and rois.  class_filter / special_assignments may be NULL with count 0.  Returns the number of exported detections. */
int mf_generate_id_image(const uint8_t* masks, int H, int W, int N, const float* scores, const int32_t* class_ids, const int32_t* rois,
                         double min_score, const int32_t* class_filter, int n_filter, const int32_t* special_assignments, int n_special,
                         uint8_t* id_image, int32_t* exported_class_ids, int32_t* exported_rois);

/* baseline JPEG -> 8-bit RGB exactly as libjpeg's default decode path produces it (islow IDCT, fancy upsampling; mf_jpeg.cu).
 * out == NULL: only the size.  Used by both loaders; exported for the decoder's own parity test. */
int mf_decode_jpeg(const uint8_t* data, int size, uint8_t* out, int capacity, int* width, int* height);

/* OpenEXR scan-line file (HALF / FLOAT channels, compression NONE / RLE / ZIPS / ZIP) -> the float depth image the -dir reader delivers:
 * what the reference keeps of cv::imread(path, IMREAD_UNCHANGED), GUI/Tools/ImageLogReader.cpp:251-258 (CV_32FC1 as is, element 0 = the
 * B channel of a CV_32FC3 result).  capacity in floats; out == NULL: only the size.  Exported for the decoder's own parity test. */
int mf_decode_exr_depth(const uint8_t* data, int size, float* out, int capacity, int* width, int* height);

/* ---- .klg log reader / writer (GUI/Tools/KlgLogReader.cpp:29-113) ---- */
typedef struct mf_klg mf_klg;
mf_klg* mf_klg_open(const char* path, int width, int height, int flip_colors);
int mf_klg_num_frames(mf_klg* k);
int mf_klg_has_more(mf_klg* k);                                         /* KlgLogReader::hasMore (N11: last frame never read) */
int mf_klg_get_next(mf_klg* k, uint8_t* rgb, float* depth, int64_t* timestamp);   /* KlgLogReader::getNext + readFrame */
void mf_klg_close(mf_klg* k);
int mf_klg_write(const char* path, int width, int height, int num_frames, const int64_t* timestamps,
                 const uint16_t* depth_mm, const uint8_t* rgb);          /* raw (uncompressed) log */

#ifdef __cplusplus
}
#endif
#endif
