// mf_sched.cu -- device-side bookkeeping of the multi-model schedule and the object-sharded exchange.
//
//   k_pack_rows / k_lifecycle   <- MaskFusion.cpp:257-276: after tracking, every tracked object whose incremental motion exceeds
//                                  0.2 m is inactivated, every static object follows the camera (Model::updateStaticPose).  The
//                                  reference takes these decisions on the host after a device sync; here one kernel reads the tracked
//                                  poses where the tracker left them (device memory), empties the stores of inactivated models (all later
//                                  passes of the frame become no-ops for them), writes the static poses, and records everything the host
//                                  wants to know in a FrameResult that is copied back asynchronously and read at the start of the NEXT frame.
//   NcclApi / ShardComm         <- SURVEY 8(e): the three couplings between object models of a frame as NCCL collectives issued from
//                                  inside the library on the context's stream (frame packet broadcast, pose-row all-gather, 64-bit MIN
//                                  all-reduce of the ID-projection keys), plus, on detector frames of a run with a detector rank, the
//                                  broadcast of that rank's frame mask and header.  libnccl is opened at run time (dlopen: the same copy torch has
//                                  already mapped, if any); a process that never shards never needs it.
#include "mf_common.cuh"
#include "mf_kernels.h"
#include "mf_host.h"
#include <dlfcn.h>
#include <string.h>

namespace mfb {

// rows of the pose table: [model][32] = pose (row-major 4x4) | last incremental transform, written by the rank that tracks the model
__global__ void k_pack_rows(LifeParams lp, float* __restrict__ table)
{
    const int i = blockIdx.x, k = threadIdx.x;                     // one block per model slot, 32 threads
    if (i >= MF_MAX_MODELS) return;
    float v = 0.f;
    if (i < lp.nModels && lp.m[i].owned && lp.m[i].tracked) v = lp.m[i].trackOut[k];
    table[i * 32 + k] = v;
}

// gathered: [world][MF_MAX_MODELS][32] (world == 1: the table itself).  One thread per model.
__global__ void k_lifecycle(LifeParams lp, const float* __restrict__ gathered, FrameResult* __restrict__ res)
{
    const int i = threadIdx.x;
    if (i >= MF_MAX_MODELS) return;
    res->dead[i] = 0; res->deadCount[i] = 0;
    if (i >= lp.nModels) return;
    const LifeModel m = lp.m[i];
    float pose[16], last[16];
    if (m.tracked) {
        const float* row = gathered + ((size_t)m.ownerRank * MF_MAX_MODELS + i) * 32;
        for (int k = 0; k < 16; ++k) { pose[k] = row[k]; last[k] = row[16 + k]; }
        const float d = sqrtf((last[3] * last[3] + last[7] * last[7]) + last[11] * last[11]);
        if (i > 0 && d > 0.2f) {                                   // inactivateModel (MaskFusion.cpp:268-272)
            res->dead[i] = 1;
            if (m.owned) { res->deadCount[i] = *m.count; *m.count = 0; }
        }
    } else {
        // Model::updateStaticPose: pose = initialC2Winv * globalPose
        mul(m.initialC2Winv, gathered, pose);                      // the background model is tracked by rank 0, slot 0
        for (int k = 0; k < 16; ++k) last[k] = (k % 5 == 0) ? 1.f : 0.f;
        if (m.owned) {
            float old[16];
            for (int k = 0; k < 12; ++k) old[k] = m.dpose->pose.m[k];
            old[12] = 0.f; old[13] = 0.f; old[14] = 0.f; old[15] = 1.f;
            derivePose(m.dpose, pose, old);                        // overridePose: lastPose = pose; pose = new
        }
    }
    for (int k = 0; k < 16; ++k) { res->poses[i][k] = pose[k]; res->poses[i][16 + k] = last[k]; }
}

void launch_pack_rows(const LifeParams& lp, float* table, Enq q) { launch(q, "k_pack_rows", k_pack_rows, MF_MAX_MODELS, 32, 0, lp, table); }
void launch_lifecycle(const LifeParams& lp, const float* gathered, FrameResult* res, Enq q)
{
    launch(q, "k_lifecycle", k_lifecycle, 1, MF_MAX_MODELS, 0, lp, gathered, res);
}
__global__ void k_set_count(uint32_t* c, uint32_t v) { if (threadIdx.x == 0 && blockIdx.x == 0) *c = v; }
void launch_set_count(uint32_t* c, uint32_t v, Enq q) { launch(q, nullptr, k_set_count, 1, 32, 0, c, v); }

// ---------------------------------------------------------------------------------------------------------------------------------
// NCCL, opened at run time.  Only the handful of entry points the exchange needs; types follow nccl.h (ABI-stable across 2.x).
// ---------------------------------------------------------------------------------------------------------------------------------
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
enum { ncclSuccess = 0 };
enum { ncclUint8 = 1, ncclUint64 = 5, ncclFloat32 = 7 };          // ncclDataType_t
enum { ncclMin = 3 };                                            // ncclRedOp_t: sum 0, prod 1, max 2, min 3

struct NcclApi {
    int (*GetUniqueId)(ncclUniqueId*) = nullptr;
    int (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    int (*CommDestroy)(ncclComm_t) = nullptr;
    int (*Broadcast)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
    int (*AllReduce)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
    int (*GetVersion)(int*) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
};
// the entry points, opened on first use (a failed open is tried again by the next call)
static const NcclApi& nccl()
{
    static const NcclApi api = [] {
        // RTLD_NOLOAD first: if the process (torch) already mapped a libnccl, use that copy; else the default search path
        void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
        if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
        if (!h) throw CudaError{std::string("object-sharded mode needs NCCL: dlopen(libnccl.so.2) failed: ") + dlerror()};
        NcclApi a;
#define MF_SYM(field, name) *(void**)(&a.field) = dlsym(h, name); if (!a.field) throw CudaError{std::string("libnccl lacks ") + name};
        MF_SYM(GetUniqueId, "ncclGetUniqueId") MF_SYM(CommInitRank, "ncclCommInitRank") MF_SYM(CommDestroy, "ncclCommDestroy")
        MF_SYM(Broadcast, "ncclBroadcast") MF_SYM(AllGather, "ncclAllGather") MF_SYM(AllReduce, "ncclAllReduce")
        MF_SYM(GetVersion, "ncclGetVersion") MF_SYM(GetErrorString, "ncclGetErrorString")
#undef MF_SYM
        return a;
    }();
    return api;
}
// r comes from an entry point, so the library is open
static void ncclCheck(int r, const char* where)
{
    if (r != ncclSuccess) throw CudaError{std::string(where) + ": " + nccl().GetErrorString(r)};
}

void shardUniqueId(unsigned char* out128)
{
    ncclUniqueId id; memset(&id, 0, sizeof id);
    ncclCheck(nccl().GetUniqueId(&id), "ncclGetUniqueId");
    memcpy(out128, id.internal, 128);
}

ShardComm::~ShardComm() { if (comm) nccl().CommDestroy((ncclComm_t)comm); }     // comm is set only once the library is open
void ShardComm::init(const unsigned char* id128, int rank_, int world_)
{
    ncclUniqueId id; memcpy(id.internal, id128, 128);
    ncclComm_t c = nullptr;
    ncclCheck(nccl().CommInitRank(&c, world_, id, rank_), "ncclCommInitRank");
    comm = c; rank = rank_; world = world_;
    int v = 0; if (nccl().GetVersion(&v) == ncclSuccess) version = v;
}
void ShardComm::broadcast(void* buf, size_t bytes, int root, cudaStream_t s)
{
    ncclCheck(nccl().Broadcast(buf, buf, bytes, ncclUint8, root, (ncclComm_t)comm, s), "ncclBroadcast (frame packet / frame masks)");
    bytesMoved += bytes; ++calls;
}
void ShardComm::allGatherFloats(const float* send, float* recv, size_t countPerRank, cudaStream_t s)
{
    ncclCheck(nccl().AllGather(send, recv, countPerRank, ncclFloat32, (ncclComm_t)comm, s), "ncclAllGather (pose rows)");
    bytesMoved += countPerRank * 4 * (size_t)world; ++calls;
}
void ShardComm::allReduceMinU64(uint64_t* buf, size_t count, cudaStream_t s)
{
    ncclCheck(nccl().AllReduce(buf, buf, count, ncclUint64, ncclMin, (ncclComm_t)comm, s), "ncclAllReduce (projection keys, 64-bit MIN)");
    bytesMoved += count * 8; ++calls;
}

}  // namespace mfb
