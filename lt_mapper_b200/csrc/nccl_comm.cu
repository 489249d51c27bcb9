// libltr_b200.so -- NCCL exchange points of the keyframe-sharded path (SURVEY.md section 8e), on the context's own stream.
//
// The path shards by keyframe (and, with two sessions, by session): every per-keyframe loop of ltremovert/src/Removerter.cpp
// and Session.cpp runs on the rank that owns the keyframe; what crosses ranks is
//   (1) the OR of the per-map-point dynamic flags of one pass (Removerter.cpp:588-590 builds the union of the per-scan index
//       sets; here each rank holds the union over ITS keyframes)          -> ncclAllReduce(uint8, max), in place;
//   (2) clouds merged over all keyframes in keyframe order (utility.cpp:177-189; contiguous keyframe blocks => rank order is
//       keyframe order)                                                    -> variable all-gather written directly in place
//       with grouped ncclSend / ncclRecv (one group for all four SoA components of all clouds of a stage);
//   (3) whole maps handed from the ranks of one session to the ranks of the other                -> ncclSend / ncclRecv pairs.
// libnccl is resolved with dlopen at first use, so single-GPU users need no NCCL at all; inside a PyTorch process the already
// loaded libnccl.so.2 (torch's) is the one that answers.
#include "ltr_internal.cuh"
#include <dlfcn.h>
#include <cstring>
#include <algorithm>

namespace ltr {

// Just the part of nccl.h this file needs (ABI-stable since NCCL 2.4; ncclCommSplit since 2.18).
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
enum { ncclSuccess = 0 };
enum { ncclInt8 = 0, ncclChar = 0, ncclUint8 = 1, ncclInt32 = 2, ncclUint32 = 3, ncclInt64 = 4, ncclUint64 = 5, ncclFloat32 = 7 };
enum { ncclSum = 0, ncclProd = 1, ncclMax = 2, ncclMin = 3 };

struct NcclApi {
    void* so = nullptr;
    int (*GetUniqueId)(ncclUniqueId*) = nullptr;
    int (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    int (*CommSplit)(ncclComm_t, int, int, ncclComm_t*, void*) = nullptr;
    int (*CommDestroy)(ncclComm_t) = nullptr;
    int (*AllReduce)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
    int (*Broadcast)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
    int (*Send)(const void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
    int (*Recv)(void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    int (*GetVersion)(int*) = nullptr;
    std::string err;
};

static NcclApi* nccl_api() {
    static NcclApi api;
    static bool tried = false;
    if (tried) return &api;
    tried = true;
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* n : names) { api.so = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (api.so) break; }
    if (!api.so) { api.err = std::string("dlopen(libnccl.so.2) failed: ") + dlerror(); return &api; }
#define LTR_SYM(field, name)                                                     \
    *(void**)(&api.field) = dlsym(api.so, name);                                  \
    if (!api.field) { api.err = std::string("libnccl lacks ") + name; api.so = nullptr; return &api; }
    LTR_SYM(GetUniqueId, "ncclGetUniqueId") LTR_SYM(CommInitRank, "ncclCommInitRank") LTR_SYM(CommSplit, "ncclCommSplit")
    LTR_SYM(CommDestroy, "ncclCommDestroy") LTR_SYM(AllReduce, "ncclAllReduce") LTR_SYM(AllGather, "ncclAllGather")
    LTR_SYM(Broadcast, "ncclBroadcast") LTR_SYM(Send, "ncclSend") LTR_SYM(Recv, "ncclRecv") LTR_SYM(GroupStart, "ncclGroupStart")
    LTR_SYM(GroupEnd, "ncclGroupEnd") LTR_SYM(GetErrorString, "ncclGetErrorString") LTR_SYM(GetVersion, "ncclGetVersion")
#undef LTR_SYM
    return &api;
}

constexpr int kMaxBatch = 16;   // clouds per grouped gather; NcclComm::h_cnt / d_cnt hold max(world, 2) * kMaxBatch slots

static std::vector<NcclComm>& comms(ltr_ctx* ctx) { return ctx->nccl; }
static inline ncclComm_t nccl_of(const NcclComm& c) { return (ncclComm_t)c.comm; }

#define LTR_NCCL(ctx, api, call)                                                                                       \
    do {                                                                                                               \
        const int r__ = (call);                                                                                        \
        if (r__ != ncclSuccess) return ::ltr::fail(ctx, LTR_ERR_CUDA, "%s failed: %s (%s:%d)", #call, (api)->GetErrorString(r__), __FILE__, __LINE__); \
    } while (0)

static int comm_get(ltr_ctx* ctx, int h, NcclComm** c) {
    auto& v = comms(ctx);
    if (h < 0 || h >= (int)v.size() || !v[h].used) return fail(ctx, LTR_ERR_INVALID, "invalid communicator handle %d", h);
    *c = &v[h];
    return LTR_OK;
}

static int comm_register(ltr_ctx* ctx, ncclComm_t nc, int rank, int world, int* out) {
    NcclComm c;
    c.comm = (void*)nc; c.rank = rank; c.world = world; c.used = true;
    LTR_CUDA(ctx, cudaMallocHost((void**)&c.h_cnt, sizeof(int64_t) * (size_t)std::max(world, 2) * kMaxBatch));
    void* p;
    LTR_TRY(dev_alloc(ctx, &p, sizeof(int64_t) * (size_t)std::max(world, 2) * kMaxBatch));
    c.d_cnt = (int64_t*)p;
    auto& v = comms(ctx);
    v.push_back(c);
    *out = (int)v.size() - 1;
    return LTR_OK;
}

int nccl_comm_info(ltr_ctx* ctx, int comm, int* rank, int* world) {
    NcclComm* c;
    LTR_TRY(comm_get(ctx, comm, &c));
    *rank = c->rank; *world = c->world;
    return LTR_OK;
}

int nccl_allreduce_u32(ltr_ctx* ctx, int comm, uint32_t* dev, size_t count, int op) {
    NcclComm* c;
    LTR_TRY(comm_get(ctx, comm, &c));
    if (c->world <= 1 || count == 0) return LTR_OK;
    NcclApi* a = nccl_api();
    LTR_NCCL(ctx, a, a->AllReduce(dev, dev, count, ncclUint32, op == 0 ? ncclSum : op == 1 ? ncclMin : ncclMax, nccl_of(*c), ctx->stream));
    return LTR_OK;
}

int nccl_alltoallv_cloud(ltr_ctx* ctx, int comm, const DevCloud& send, const std::vector<int64_t>& scount, CloudOwner* recv_out) {
    NcclComm* cp;
    LTR_TRY(comm_get(ctx, comm, &cp));
    const NcclComm cc = *cp;
    const int G = cc.world;
    if ((int)scount.size() != G || G > 16) return fail(ctx, LTR_ERR_INVALID, "alltoallv: bad count vector");
    std::vector<int64_t> all((size_t)G * G);
    LTR_TRY(ltr_nccl_allgather_i64(ctx, comm, scount.data(), G, all.data()));   // all[r * G + d] = points rank r sends to rank d
    std::vector<int64_t> sdispl((size_t)G + 1, 0), rdispl((size_t)G + 1, 0);
    for (int d = 0; d < G; ++d) sdispl[d + 1] = sdispl[d] + scount[d];
    for (int r = 0; r < G; ++r) rdispl[r + 1] = rdispl[r] + all[(size_t)r * G + cc.rank];
    LTR_TRY(cloud_new(ctx, rdispl[G], recv_out));
    const DevCloud dst = ctx->clouds[recv_out->get()];
    const float* sp[4] = {send.x(), send.y(), send.z(), send.i()};
    float* dp[4] = {dst.x(), dst.y(), dst.z(), dst.i()};
    NcclApi* a = nccl_api();
    LTR_NCCL(ctx, a, a->GroupStart());
    for (int r = 0; r < G; ++r) {
        if (r == cc.rank) continue;
        const int64_t ns = scount[r], nr = all[(size_t)r * G + cc.rank];
        for (int k = 0; k < 4; ++k) {
            if (ns > 0) LTR_NCCL(ctx, a, a->Send(sp[k] + sdispl[r], (size_t)ns, ncclFloat32, r, nccl_of(cc), ctx->stream));
            if (nr > 0) LTR_NCCL(ctx, a, a->Recv(dp[k] + rdispl[r], (size_t)nr, ncclFloat32, r, nccl_of(cc), ctx->stream));
        }
    }
    LTR_NCCL(ctx, a, a->GroupEnd());
    if (scount[cc.rank] > 0)
        for (int k = 0; k < 4; ++k)
            LTR_CUDA(ctx, cudaMemcpyAsync(dp[k] + rdispl[cc.rank], sp[k] + sdispl[cc.rank], (size_t)scount[cc.rank] * sizeof(float), cudaMemcpyDeviceToDevice, ctx->stream));
    return LTR_OK;
}

}  // namespace ltr

using namespace ltr;

extern "C" {

int ltr_nccl_unique_id(uint8_t* id128) {
    NcclApi* a = nccl_api();
    if (!a->so) { g_create_err = a->err; return LTR_ERR_CUDA; }
    ncclUniqueId id;
    const int r = a->GetUniqueId(&id);
    if (r != ncclSuccess) { g_create_err = a->GetErrorString(r); return LTR_ERR_CUDA; }
    std::memcpy(id128, id.internal, 128);
    return LTR_OK;
}

int ltr_nccl_init(ltr_ctx* ctx, const uint8_t* id128, int32_t rank, int32_t world, int32_t* comm_out) {
    if (!ctx || !id128 || !comm_out || world < 1 || rank < 0 || rank >= world) return fail(ctx, LTR_ERR_INVALID, "bad argument");
    NcclApi* a = nccl_api();
    if (!a->so) return fail(ctx, LTR_ERR_CUDA, "%s", a->err.c_str());
    LTR_CUDA(ctx, cudaSetDevice(ctx->device));
    ncclUniqueId id;
    std::memcpy(id.internal, id128, 128);
    ncclComm_t nc = nullptr;
    LTR_NCCL(ctx, a, a->CommInitRank(&nc, world, id, rank));
    return comm_register(ctx, nc, rank, world, comm_out);
}

int ltr_nccl_split(ltr_ctx* ctx, int32_t comm, int32_t color, int32_t key, int32_t* comm_out) {
    ApiTrace tr__(ctx, "ltr_nccl_split");
    NcclComm* c;
    LTR_TRY(comm_get(ctx, comm, &c));
    NcclApi* a = nccl_api();
    ncclComm_t nc = nullptr;
    const NcclComm parent = *c;
    LTR_NCCL(ctx, a, a->CommSplit(nccl_of(parent), color, key, &nc, nullptr));
    // ranks inside the new communicator are ordered by key; the caller passes key == parent rank and equal-sized colours
    int members = 0, myrank = 0;
    {   // count members of my colour through the parent (one small all-gather of (color, key))
        int64_t* h = parent.h_cnt; int64_t* d = parent.d_cnt;
        h[0] = ((int64_t)color << 32) | (uint32_t)key;
        LTR_CUDA(ctx, cudaMemcpyAsync(d + parent.rank, h, sizeof(int64_t), cudaMemcpyHostToDevice, ctx->stream));
        LTR_NCCL(ctx, a, a->AllGather(d + parent.rank, d, 1, ncclInt64, nccl_of(parent), ctx->stream));
        LTR_CUDA(ctx, cudaMemcpyAsync(h, d, sizeof(int64_t) * (size_t)parent.world, cudaMemcpyDeviceToHost, ctx->stream));
        LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        for (int r = 0; r < parent.world; ++r)
            if ((int32_t)(h[r] >> 32) == color) { ++members; if ((int32_t)(uint32_t)h[r] < key) ++myrank; }
    }
    return comm_register(ctx, nc, myrank, members, comm_out);
}

int ltr_nccl_info(ltr_ctx* ctx, int32_t comm, int32_t* rank, int32_t* world) {
    NcclComm* c;
    LTR_TRY(comm_get(ctx, comm, &c));
    if (rank) *rank = c->rank;
    if (world) *world = c->world;
    return LTR_OK;
}

int ltr_nccl_destroy(ltr_ctx* ctx, int32_t comm) {
    ApiTrace tr__(ctx, "ltr_nccl_destroy");
    NcclComm* c;
    LTR_TRY(comm_get(ctx, comm, &c));
    cudaStreamSynchronize(ctx->stream);
    nccl_api()->CommDestroy(nccl_of(*c));
    cudaFreeHost(c->h_cnt);
    dev_free(ctx, c->d_cnt);
    *c = NcclComm();
    return LTR_OK;
}

int ltr_nccl_version(int32_t* v) {
    NcclApi* a = nccl_api();
    if (!a->so) return LTR_ERR_CUDA;
    int x = 0;
    a->GetVersion(&x);
    *v = x;
    return LTR_OK;
}

// (1) flag union: in-place max-reduction of the N dynamic-flag bytes of `map` (every rank holds the same map)
int ltr_nccl_allreduce_flags(ltr_ctx* ctx, int32_t comm, ltr_cloud map) {
    ApiTrace tr__(ctx, "ltr_nccl_allreduce_flags");
    NcclComm* c;
    DevCloud* m;
    LTR_TRY(comm_get(ctx, comm, &c));
    LTR_TRY(cloud_get(ctx, map, &m));
    if (c->world <= 1 || m->n == 0) return LTR_OK;
    LTR_TRY(cloud_ensure_flags(ctx, m));
    NcclApi* a = nccl_api();
    LTR_NCCL(ctx, a, a->AllReduce(m->flags, m->flags, (size_t)m->n, ncclUint8, ncclMax, nccl_of(*c), ctx->stream));
    return LTR_OK;
}

int ltr_nccl_allgather_i64(ltr_ctx* ctx, int32_t comm, const int64_t* local, int32_t count, int64_t* out /* world*count */) {
    ApiTrace tr__(ctx, "ltr_nccl_allgather_i64");
    NcclComm* c;
    LTR_TRY(comm_get(ctx, comm, &c));
    if (count < 1 || count > kMaxBatch) return fail(ctx, LTR_ERR_INVALID, "count %d outside [1, %d]", count, kMaxBatch);
    if (c->world <= 1) { std::memcpy(out, local, sizeof(int64_t) * (size_t)count); return LTR_OK; }
    NcclApi* a = nccl_api();
    std::memcpy(c->h_cnt, local, sizeof(int64_t) * (size_t)count);
    int64_t* mine = c->d_cnt + (size_t)c->rank * count;
    LTR_CUDA(ctx, cudaMemcpyAsync(mine, c->h_cnt, sizeof(int64_t) * (size_t)count, cudaMemcpyHostToDevice, ctx->stream));
    LTR_NCCL(ctx, a, a->AllGather(mine, c->d_cnt, (size_t)count, ncclInt64, nccl_of(*c), ctx->stream));
    LTR_CUDA(ctx, cudaMemcpyAsync(c->h_cnt, c->d_cnt, sizeof(int64_t) * (size_t)count * c->world, cudaMemcpyDeviceToHost, ctx->stream));
    LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    std::memcpy(out, c->h_cnt, sizeof(int64_t) * (size_t)count * c->world);
    return LTR_OK;
}

// (2) rank-ordered variable all-gather of `count` clouds at once: out[i] = concat over ranks r = 0..world-1 of rank r's local[i].
// One count exchange for all clouds, then ONE NCCL group that moves every SoA component of every cloud directly into place.
int ltr_nccl_allgather_clouds(ltr_ctx* ctx, int32_t comm, int32_t count, const ltr_cloud* local, ltr_cloud* out) {
    ApiTrace tr__(ctx, "ltr_nccl_allgather_clouds");
    NcclComm* c;
    LTR_TRY(comm_get(ctx, comm, &c));
    if (!local || !out || count < 1 || count > kMaxBatch) return fail(ctx, LTR_ERR_INVALID, "bad argument");
    const NcclComm cc = *c;
    std::vector<CloudOwner> o((size_t)count);
    if (cc.world <= 1) {
        for (int i = 0; i < count; ++i) {
            ltr_cloud h;
            LTR_TRY(ltr_cloud_copy(ctx, local[i], &h));
            o[i] = CloudOwner(ctx, h);
        }
        for (int i = 0; i < count; ++i) out[i] = o[i].release();
        return LTR_OK;
    }
    int64_t mine[kMaxBatch];
    for (int i = 0; i < count; ++i) { DevCloud* l; LTR_TRY(cloud_get(ctx, local[i], &l)); mine[i] = l->n; }
    std::vector<int64_t> all((size_t)cc.world * count);
    LTR_TRY(ltr_nccl_allgather_i64(ctx, comm, mine, count, all.data()));
    NcclApi* a = nccl_api();
    std::vector<std::vector<int64_t>> displs((size_t)count, std::vector<int64_t>((size_t)cc.world + 1, 0));
    for (int i = 0; i < count; ++i) {
        for (int r = 0; r < cc.world; ++r) displs[i][r + 1] = displs[i][r] + all[(size_t)r * count + i];
        LTR_TRY(cloud_new(ctx, displs[i][cc.world], &o[i]));
    }
    LTR_NCCL(ctx, a, a->GroupStart());
    for (int i = 0; i < count; ++i) {
        const DevCloud src = ctx->clouds[local[i]];
        const DevCloud dst = ctx->clouds[o[i].get()];
        const float* sp[4] = {src.x(), src.y(), src.z(), src.i()};
        float* dp[4] = {dst.x(), dst.y(), dst.z(), dst.i()};
        for (int r = 0; r < cc.world; ++r) {
            if (r == cc.rank) continue;
            const int64_t nr = all[(size_t)r * count + i];
            for (int k = 0; k < 4; ++k) {
                if (src.n > 0) LTR_NCCL(ctx, a, a->Send(sp[k], (size_t)src.n, ncclFloat32, r, nccl_of(cc), ctx->stream));
                if (nr > 0) LTR_NCCL(ctx, a, a->Recv(dp[k] + displs[i][r], (size_t)nr, ncclFloat32, r, nccl_of(cc), ctx->stream));
            }
        }
    }
    LTR_NCCL(ctx, a, a->GroupEnd());
    for (int i = 0; i < count; ++i) {
        const DevCloud src = ctx->clouds[local[i]];
        const DevCloud dst = ctx->clouds[o[i].get()];
        if (src.n > 0)
            LTR_CUDA(ctx, cudaMemcpy2DAsync(dst.base + displs[i][cc.rank], (size_t)dst.cap * 4, src.base, (size_t)src.cap * 4, (size_t)src.n * 4, 4,
                                            cudaMemcpyDeviceToDevice, ctx->stream));
    }
    for (int i = 0; i < count; ++i) out[i] = o[i].release();
    return LTR_OK;
}

// (3) hand whole clouds to / take whole clouds from one peer: n_send clouds go to `peer`, n_recv clouds come from `peer`
// (both sides call with mirrored counts).  Sizes travel first (one grouped send/recv of the counts), then one group for the data.
int ltr_nccl_exchange_clouds(ltr_ctx* ctx, int32_t comm, int32_t peer, int32_t n_send, const ltr_cloud* send, int32_t n_recv, ltr_cloud* recv) {
    ApiTrace tr__(ctx, "ltr_nccl_exchange_clouds");
    NcclComm* c;
    LTR_TRY(comm_get(ctx, comm, &c));
    const NcclComm cc = *c;
    if (peer < 0 || peer >= cc.world || peer == cc.rank) return fail(ctx, LTR_ERR_INVALID, "bad peer %d", peer);
    if (n_send < 0 || n_recv < 0 || n_send > kMaxBatch || n_recv > kMaxBatch) return fail(ctx, LTR_ERR_INVALID, "bad counts");
    NcclApi* a = nccl_api();
    int64_t* h = cc.h_cnt;
    int64_t* d = cc.d_cnt;                 // [0, n_send): my sizes, [kMaxBatch, kMaxBatch + n_recv): the peer's  (world >= 2 => 2 * kMaxBatch slots exist)
    for (int i = 0; i < n_send; ++i) { DevCloud* s; LTR_TRY(cloud_get(ctx, send[i], &s)); h[i] = s->n; }
    if (n_send > 0) LTR_CUDA(ctx, cudaMemcpyAsync(d, h, sizeof(int64_t) * (size_t)n_send, cudaMemcpyHostToDevice, ctx->stream));
    LTR_NCCL(ctx, a, a->GroupStart());
    if (n_send > 0) LTR_NCCL(ctx, a, a->Send(d, (size_t)n_send, ncclInt64, peer, nccl_of(cc), ctx->stream));
    if (n_recv > 0) LTR_NCCL(ctx, a, a->Recv(d + kMaxBatch, (size_t)n_recv, ncclInt64, peer, nccl_of(cc), ctx->stream));
    LTR_NCCL(ctx, a, a->GroupEnd());
    if (n_recv > 0) LTR_CUDA(ctx, cudaMemcpyAsync(h + kMaxBatch, d + kMaxBatch, sizeof(int64_t) * (size_t)n_recv, cudaMemcpyDeviceToHost, ctx->stream));
    // also on a send-only side: the pinned staging slots h[0, n_send) are reused by the next count exchange on this communicator,
    // which must not overwrite them before the asynchronous upload above has read them
    LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    std::vector<CloudOwner> o((size_t)n_recv);
    for (int i = 0; i < n_recv; ++i) LTR_TRY(cloud_new(ctx, h[kMaxBatch + i], &o[i]));
    LTR_NCCL(ctx, a, a->GroupStart());
    for (int i = 0; i < n_send; ++i) {
        const DevCloud s = ctx->clouds[send[i]];
        const float* sp[4] = {s.x(), s.y(), s.z(), s.i()};
        if (s.n > 0) for (int k = 0; k < 4; ++k) LTR_NCCL(ctx, a, a->Send(sp[k], (size_t)s.n, ncclFloat32, peer, nccl_of(cc), ctx->stream));
    }
    for (int i = 0; i < n_recv; ++i) {
        const DevCloud r = ctx->clouds[o[i].get()];
        float* rp[4] = {r.x(), r.y(), r.z(), r.i()};
        if (r.n > 0) for (int k = 0; k < 4; ++k) LTR_NCCL(ctx, a, a->Recv(rp[k], (size_t)r.n, ncclFloat32, peer, nccl_of(cc), ctx->stream));
    }
    LTR_NCCL(ctx, a, a->GroupEnd());
    for (int i = 0; i < n_recv; ++i) recv[i] = o[i].release();
    return LTR_OK;
}

// max over ranks of one double (timings), via an all-gather of the raw bits
int ltr_nccl_max_f64(ltr_ctx* ctx, int32_t comm, double v, double* out) {
    NcclComm* c;
    LTR_TRY(comm_get(ctx, comm, &c));
    std::vector<int64_t> all((size_t)c->world);
    int64_t bits;
    std::memcpy(&bits, &v, 8);
    LTR_TRY(ltr_nccl_allgather_i64(ctx, comm, &bits, 1, all.data()));
    double m = v;
    for (int64_t b : all) { double x; std::memcpy(&x, &b, 8); if (x > m) m = x; }
    *out = m;
    return LTR_OK;
}

int ltr_nccl_barrier(ltr_ctx* ctx, int32_t comm) {
    int64_t z = 0;
    NcclComm* c;
    LTR_TRY(comm_get(ctx, comm, &c));
    std::vector<int64_t> all((size_t)c->world);
    return ltr_nccl_allgather_i64(ctx, comm, &z, 1, all.data());
}

}  // extern "C"
