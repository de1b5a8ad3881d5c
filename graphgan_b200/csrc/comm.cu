// comm.cu -- the data-parallel optimizer step with its collective INSIDE the library (sm_90a + NCCL over NVLink).
//
// Data parallelism: partition the root set over the GPUs of one NVLink box, with a single NCCL collective of the
// embedding gradients per step.  The reference has no collective at all; the call sites this replaces
// are the per-batch sess.run loops of graph_gan.py:149-157 / 168-176, run on N replicas.
//
//   every rank:  K2 on ITS slice of the mini-batch  ->  ONE ncclAllGather of the compact gradients
//                (rows[cap, ld] | bias[cap] | ids[cap] | n_unique: a few KB -- latency bound, which NVSwitch is good at)
//                ->  deterministic rank-major merge (gg_grad_merge)  ->  the same K3 sweep on every rank.
//
// Above GG_MAX_BATCH pairs (gg_dp_step_ex / gg_dp_train_steps_ex, NCCL only) the slice gradient and the merge are the
// multi-CTA gg_pair_grad_ex and gg_grad_merge_ex (grad_multi.cu), with the same entry order and sums.
//
// An all-gather + ordered merge instead of a float all-reduce: (i) the dense [N, ld] gradient is 512 MB per step at
// C3 against 64 KB compact, and (ii) every replica adds the same floats in the same order, so replicas stay
// BIT-IDENTICAL without ever broadcasting parameters.  All four stages are enqueued on the caller's stream from C
// (gg_dp_train_steps walks a whole shuffled start list): no host-language round trip and no synchronisation per step.
//
// NCCL is resolved at run time: dlopen("libnccl.so.2", RTLD_NOLOAD) first, so that inside a PyTorch process the
// library shares torch's own NCCL (two NCCL copies in one process is the thing to avoid); a plain dlopen otherwise.
// The library still loads, and everything else works, on a machine without NCCL.
#include <dlfcn.h>
#include <math.h>
#include <string.h>

#include "update_dev.cuh"

namespace gg {
namespace {

// the slice of the NCCL ABI used here (stable since NCCL 2.0)
typedef struct ncclComm *ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
typedef int ncclResult_t;                 // ncclSuccess == 0
constexpr int NCCL_FLOAT32 = 7;           // ncclFloat32 in ncclDataType_t

struct NcclApi {
    void *handle = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllGather)(const void *, void *, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GetVersion)(int *) = nullptr;
    const char *(*GetErrorString)(ncclResult_t) = nullptr;
    bool ok = false;
};

NcclApi &nccl() {
    static NcclApi api;
    if (api.handle) return api;
    void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);      // torch's copy, when it is already in the process
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return api;
    api.handle = h;
    api.GetUniqueId = (decltype(api.GetUniqueId))dlsym(h, "ncclGetUniqueId");
    api.CommInitRank = (decltype(api.CommInitRank))dlsym(h, "ncclCommInitRank");
    api.CommDestroy = (decltype(api.CommDestroy))dlsym(h, "ncclCommDestroy");
    api.AllGather = (decltype(api.AllGather))dlsym(h, "ncclAllGather");
    api.GetVersion = (decltype(api.GetVersion))dlsym(h, "ncclGetVersion");
    api.GetErrorString = (decltype(api.GetErrorString))dlsym(h, "ncclGetErrorString");
    api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.AllGather && api.GetErrorString;
    return api;
}

int check_nccl(ncclResult_t r, const char *what) {
    if (r == 0) return 0;
    set_error("NCCL error %d (%s) at %s", (int)r, nccl().GetErrorString ? nccl().GetErrorString(r) : "?", what);
    return 3;
}

struct Comm {
    ncclComm_t comm;
    int rank, world;
    unsigned long long collectives;       // NCCL collectives issued through this handle (diagnostic, read by gg_comm_info)
    // ---- optional peer-memory transport (gg_comm_p2p_*): every rank owns an exchange buffer that all peers map
    // through CUDA IPC; the gradient kernel itself stores this rank's compact gradient into every peer's buffer
    // over NVLink and raises a flag there, the merge kernel waits for the flags -- no collective call in the step
    float *xbuf;                          // this rank's exchange buffer: [2][capacity] floats + [2][world] flags
    long long capacity;                   // floats per parity half
    float **peers_dev;                    // device array [world]: every rank's xbuf as mapped in THIS process
    void *peer_map[64];                   // host copies (for cudaIpcCloseMemHandle)
    unsigned step;                        // steps pushed so far (flag value of the next step = step + 1)
    unsigned long long p2p_steps;
    bool p2p;
};

// ---------------------------------------------------------------- fused gradient + exchange (peer memory)
__device__ __forceinline__ void st_release_sys(unsigned *p, unsigned v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned *p) {
    unsigned v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

// K2 on this rank's slice of the mini-batch, then -- in the same kernel -- the exchange: the compact gradient (nf
// floats) is stored into slot `rank` of EVERY rank's exchange buffer (peer stores over NVLink, 16 bytes per thread
// per instruction) and, after a system-scope fence, a release store of the step number into that rank's flag word.
__global__ void __launch_bounds__(GRAD_THREADS, 1)
pair_grad_push_kernel(int mode, int B, int batch_total, const int *__restrict__ ni, const int *__restrict__ nj,
                      const float *__restrict__ aux, const float *__restrict__ emb, const float *__restrict__ bias, int ld,
                      float lambda, float *local_buf, int cap, int *row_slot, float *const *__restrict__ peers, int rank,
                      int world, long long capacity, unsigned step_id) {
    extern __shared__ int smem[];
    const int tid = threadIdx.x;
    const long long nf = (long long)cap * ld + 2ll * cap + 4;
    float *rows_p = local_buf, *bias_p = local_buf + (size_t)cap * ld;
    int *ids_p = reinterpret_cast<int *>(bias_p + cap), *nu_p = ids_p + cap;
    if (B > 0) {
        pair_grad_body<false>(smem, mode, B, batch_total, ni, nj, aux, emb, bias, ld, lambda, nu_p, ids_p, rows_p, bias_p, row_slot);
    } else if (tid == 0) {
        *nu_p = 0;
    }
    __threadfence();
    __syncthreads();
    const unsigned parity = step_id & 1u;
    const int nu = *nu_p;                                      // only the used slots travel: rows [0, nu) + the tail
    const long long tail0 = (long long)cap * ld;               // bias | ids | n_unique
    const long long nrow4 = ((long long)nu * ld) >> 2, ntail4 = (nf - tail0) >> 2;
    for (int r = 0; r < world; ++r) {
        float *dst = peers[r] + (size_t)parity * (size_t)capacity + (size_t)rank * (size_t)nf;
        const float4 *src4 = reinterpret_cast<const float4 *>(local_buf);
        float4 *dst4 = reinterpret_cast<float4 *>(dst);
        for (long long i = tid; i < nrow4; i += GRAD_THREADS) dst4[i] = src4[i];
        for (long long i = tid; i < ntail4; i += GRAD_THREADS) dst4[(tail0 >> 2) + i] = src4[(tail0 >> 2) + i];
    }
    __threadfence_system();
    __syncthreads();
    if (tid < world) {
        unsigned *flags = reinterpret_cast<unsigned *>(peers[tid] + 2 * (size_t)capacity);
        st_release_sys(flags + parity * world + rank, step_id);
    }
}

// waits until every rank's gradient of step `step_id` has landed in THIS rank's exchange buffer, then the rank-major merge
__global__ void __launch_bounds__(MERGE_THREADS, 1)
merge_wait_kernel(int world, int cap, int ld, const float *xbuf, long long capacity, unsigned step_id, int *__restrict__ n_unique,
                  int *__restrict__ uniq_ids, float *__restrict__ grad_rows, float *__restrict__ grad_bias,
                  int *__restrict__ row_slot) {
    extern __shared__ int smem[];
    const unsigned parity = step_id & 1u;
    if ((int)threadIdx.x < world) {
        const unsigned *flag = reinterpret_cast<const unsigned *>(xbuf + 2 * (size_t)capacity) + parity * world + threadIdx.x;
        while (ld_acquire_sys(flag) != step_id) __nanosleep(20);
    }
    __syncthreads();
    grad_merge_body(smem, world, cap, ld, xbuf + (size_t)parity * (size_t)capacity, n_unique, uniq_ids, grad_rows, grad_bias, row_slot);
}

}  // namespace
}  // namespace gg

#define GG_NCCL(call)                                       \
    do {                                                    \
        int _rc = gg::check_nccl((call), #call);            \
        if (_rc) return _rc;                                \
    } while (0)

extern "C" int gg_comm_unique_id(void *id128) {
    GG_REQUIRE(id128, "null pointer");
    gg::NcclApi &n = gg::nccl();
    GG_REQUIRE(n.ok, "libnccl.so.2 not found (dlopen)");
    gg::ncclUniqueId id;
    GG_NCCL(n.GetUniqueId(&id));
    memcpy(id128, &id, sizeof(id));
    return 0;
}

extern "C" int gg_comm_init(const void *id128, int32_t rank, int32_t world, void **comm_out) {
    GG_REQUIRE(id128 && comm_out && world >= 1 && rank >= 0 && rank < world, "bad arguments");
    gg::NcclApi &n = gg::nccl();
    GG_REQUIRE(n.ok, "libnccl.so.2 not found (dlopen)");
    gg::ncclUniqueId id;
    memcpy(&id, id128, sizeof(id));
    gg::Comm *c = new gg::Comm();
    c->comm = nullptr; c->rank = rank; c->world = world; c->collectives = 0ull;
    c->xbuf = nullptr; c->capacity = 0; c->peers_dev = nullptr; c->step = 0u; c->p2p_steps = 0ull; c->p2p = false;
    for (int i = 0; i < 64; ++i) c->peer_map[i] = nullptr;
    int rc = gg::check_nccl(n.CommInitRank(&c->comm, world, id, rank), "ncclCommInitRank");
    if (rc) { delete c; return rc; }
    *comm_out = c;
    return 0;
}

extern "C" int gg_comm_destroy(void *comm) {
    if (!comm) return 0;
    gg::Comm *c = (gg::Comm *)comm;
    for (int r = 0; r < c->world && r < 64; ++r)
        if (c->peer_map[r] && r != c->rank) cudaIpcCloseMemHandle(c->peer_map[r]);
    if (c->peers_dev) cudaFree(c->peers_dev);
    if (c->xbuf) cudaFree(c->xbuf);
    int rc = c->comm ? gg::check_nccl(gg::nccl().CommDestroy(c->comm), "ncclCommDestroy") : 0;
    delete c;
    return rc;
}

extern "C" int gg_comm_info(void *comm, int32_t *rank, int32_t *world, int32_t *nccl_version, uint64_t *collectives) {
    GG_REQUIRE(comm, "null communicator");
    gg::Comm *c = (gg::Comm *)comm;
    if (rank) *rank = c->rank;
    if (world) *world = c->world;
    if (collectives) *collectives = c->collectives + c->p2p_steps;
    if (nccl_version) {
        int v = 0;
        if (gg::nccl().GetVersion) gg::nccl().GetVersion(&v);
        *nccl_version = v;
    }
    return 0;
}

extern "C" int gg_comm_p2p_export(void *comm, int64_t capacity_floats, void *handle64) {
    GG_REQUIRE(comm && handle64 && capacity_floats > 0, "bad arguments");
    gg::Comm *c = (gg::Comm *)comm;
    GG_REQUIRE(c->world <= 64, "at most 64 ranks");
    GG_REQUIRE(!c->xbuf, "exchange buffer already created");
    const long long cap4 = (capacity_floats + 3) & ~3ll;
    const size_t bytes = (size_t)(2 * cap4 + 2 * c->world + 4) * 4;
    GG_CHECK(cudaMalloc((void **)&c->xbuf, bytes));
    GG_CHECK(cudaMemset(c->xbuf, 0, bytes));
    c->capacity = cap4;
    cudaIpcMemHandle_t h;
    GG_CHECK(cudaIpcGetMemHandle(&h, c->xbuf));
    static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
    memcpy(handle64, &h, 64);
    return 0;
}

extern "C" int gg_comm_p2p_connect(void *comm, const void *all_handles) {
    GG_REQUIRE(comm && all_handles, "bad arguments");
    gg::Comm *c = (gg::Comm *)comm;
    GG_REQUIRE(c->xbuf, "gg_comm_p2p_export first");
    float *host_ptrs[64];
    for (int r = 0; r < c->world; ++r) {
        if (r == c->rank) { host_ptrs[r] = c->xbuf; c->peer_map[r] = c->xbuf; continue; }
        cudaIpcMemHandle_t h;
        memcpy(&h, (const char *)all_handles + 64 * (size_t)r, 64);
        void *p = nullptr;
        GG_CHECK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
        c->peer_map[r] = p;
        host_ptrs[r] = (float *)p;
    }
    GG_CHECK(cudaMalloc((void **)&c->peers_dev, sizeof(float *) * (size_t)c->world));
    GG_CHECK(cudaMemcpy(c->peers_dev, host_ptrs, sizeof(float *) * (size_t)c->world, cudaMemcpyHostToDevice));
    c->p2p = true;
    return 0;
}

extern "C" int gg_comm_use_p2p(void *comm, int32_t on) {
    GG_REQUIRE(comm, "null communicator");
    gg::Comm *c = (gg::Comm *)comm;
    GG_REQUIRE(!on || c->peers_dev, "peer memory is not connected (gg_comm_p2p_export / gg_comm_p2p_connect)");
    c->p2p = on != 0;
    return 0;
}

// rows [lo, hi) of a batch of `total` rows owned by `rank` (contiguous blocks, sizes differ by at most one)
static void block_range(int total, int rank, int world, int *lo, int *hi) {
    const int base = total / world, rem = total % world;
    *lo = rank * base + (rank < rem ? rank : rem);
    *hi = *lo + base + (rank < rem ? 1 : 0);
}

extern "C" int gg_dp_step(void *comm, int32_t mode, int32_t n_pairs, const int32_t *node_id, const int32_t *node_neighbor_id,
                          const float *aux, int64_t n_node, int32_t ld, float *emb, float *m_emb, float *v_emb, float *bias,
                          float *m_bias, float *v_bias, float lambda, float *local_buf, float *gathered_buf, int32_t cap,
                          int32_t *n_unique, int32_t *uniq_ids, float *grad_rows, float *grad_bias, int32_t *row_slot,
                          float lr_t, float beta1, float beta2, float eps, void *stream) {
    GG_REQUIRE(comm, "null communicator");
    GG_REQUIRE(node_id && node_neighbor_id && aux && local_buf && gathered_buf, "null pointer");
    gg::Comm *c = (gg::Comm *)comm;
    GG_REQUIRE(n_pairs > 0 && n_pairs <= GG_MAX_BATCH, "batch size out of range");
    GG_REQUIRE(cap >= 2 * ((n_pairs + c->world - 1) / c->world), "cap too small: need 2 * ceil(n_pairs / world)");
    cudaStream_t st = (cudaStream_t)stream;
    int lo, hi;
    block_range(n_pairs, c->rank, c->world, &lo, &hi);
    const int64_t nf = gg_grad_buf_floats(cap, ld);
    if (c->p2p) {
        // ---- peer-memory transport: gradient + exchange in ONE kernel (stores into every peer's buffer over NVLink),
        // then the merge kernel waits for all ranks' flags of this step
        GG_REQUIRE((int64_t)c->world * nf <= c->capacity, "exchange buffer too small for this cap / ld");
        GG_REQUIRE(mode == 0 || mode == 1, "mode must be 0 (discriminator) or 1 (generator)");
        GG_REQUIRE(gg::ld_supported(ld), GG_LD_MESSAGE);
        const unsigned step_id = ++c->step;
        const int B = hi - lo;
        const size_t smem_g = gg::pair_grad_smem_bytes(B > 0 ? B : 1);
        gg::pair_grad_push_kernel<<<1, gg::GRAD_THREADS, smem_g, st>>>(mode, B, n_pairs, node_id + lo, node_neighbor_id + lo, aux + lo, emb,
                                                                      bias, ld, lambda, local_buf, cap, row_slot, c->peers_dev, c->rank,
                                                                      c->world, c->capacity, step_id);
        GG_CHECK(cudaGetLastError());
        const size_t smem_m = (size_t)c->world * cap * 2 * 4;
        GG_REQUIRE(smem_m <= 200 * 1024, "merge exceeds shared memory");
        if (smem_m > 48 * 1024)
            GG_CHECK(cudaFuncSetAttribute(gg::merge_wait_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_m));
        gg::merge_wait_kernel<<<1, gg::MERGE_THREADS, smem_m, st>>>(c->world, cap, ld, c->xbuf, c->capacity, step_id, n_unique, uniq_ids,
                                                                   grad_rows, grad_bias, row_slot);
        GG_CHECK(cudaGetLastError());
        c->p2p_steps += 1;
        return gg_adam_apply(n_node, ld, emb, m_emb, v_emb, bias, m_bias, v_bias, n_unique, uniq_ids, grad_rows, grad_bias, row_slot,
                             lr_t, beta1, beta2, eps, stream);
    }
    float *rows_p = local_buf, *bias_p = local_buf + (size_t)cap * ld;
    int32_t *ids_p = (int32_t *)(bias_p + cap), *nu_p = ids_p + cap;
    if (hi > lo) {      // K2 on this rank's slice; the generator loss is a mean over the WHOLE batch (batch_total)
        int rc = gg_pair_grad(mode, hi - lo, n_pairs, node_id + lo, node_neighbor_id + lo, aux + lo, emb, bias, ld, lambda, nu_p,
                              ids_p, rows_p, bias_p, row_slot, stream);
        if (rc) return rc;
    } else {
        GG_CHECK(cudaMemsetAsync(nu_p, 0, sizeof(float) * (size_t)(nf - ((size_t)cap * ld + 2 * (size_t)cap)), st));
    }
    GG_NCCL(gg::nccl().AllGather(local_buf, gathered_buf, (size_t)nf, gg::NCCL_FLOAT32, c->comm, st));   // the step's only collective
    c->collectives += 1;
    int rc = gg_grad_merge(c->world, cap, ld, gathered_buf, n_unique, uniq_ids, grad_rows, grad_bias, row_slot, stream);
    if (rc) return rc;
    return gg_adam_apply(n_node, ld, emb, m_emb, v_emb, bias, m_bias, v_bias, n_unique, uniq_ids, grad_rows, grad_bias, row_slot,
                         lr_t, beta1, beta2, eps, stream);
}

extern "C" int gg_dp_train_steps(void *comm, int32_t mode, int64_t n_rows, const int64_t *start_list, int64_t n_starts,
                                 int32_t batch_size, const int32_t *node_id, const int32_t *node_neighbor_id, const float *aux,
                                 int64_t n_node, int32_t ld, float *emb, float *m_emb, float *v_emb, float *bias, float *m_bias,
                                 float *v_bias, float lambda, float *local_buf, float *gathered_buf, int32_t cap,
                                 int32_t *n_unique, int32_t *uniq_ids, float *grad_rows, float *grad_bias, int32_t *row_slot,
                                 float lr, float beta1, float beta2, float eps, float *beta1_power, float *beta2_power,
                                 void *stream) {
    GG_REQUIRE(start_list && beta1_power && beta2_power, "null host pointer");
    GG_REQUIRE(batch_size > 0 && batch_size <= GG_MAX_BATCH, "batch size out of range");
    for (int64_t s = 0; s < n_starts; ++s) {
        const int64_t start = start_list[s];
        GG_REQUIRE(start >= 0 && start < n_rows, "start out of range");
        const int64_t end = start + batch_size < n_rows ? start + batch_size : n_rows;
        // lr_t = lr * sqrt(1 - beta2^t) / (1 - beta1^t), fp32 step by step like the TF graph (== gg_train_steps)
        volatile float one_m_b2 = 1.0f - *beta2_power;
        volatile float root = sqrtf(one_m_b2);
        volatile float num = lr * root;
        volatile float den = 1.0f - *beta1_power;
        const float lr_t = num / den;
        int rc = gg_dp_step(comm, mode, (int32_t)(end - start), node_id + start, node_neighbor_id + start, aux + start, n_node, ld,
                            emb, m_emb, v_emb, bias, m_bias, v_bias, lambda, local_buf, gathered_buf, cap, n_unique, uniq_ids,
                            grad_rows, grad_bias, row_slot, lr_t, beta1, beta2, eps, stream);
        if (rc) return rc;
        volatile float p1 = *beta1_power * beta1, p2 = *beta2_power * beta2;
        *beta1_power = p1;
        *beta2_power = p2;
    }
    return 0;
}

// ---------------------------------------------------------------- the same step for any batch size
// Slice gradient (gg_pair_grad_ex: one CTA up to GG_MAX_BATCH pairs, multi-CTA above), the same single ncclAllGather, the
// multi-CTA merge (gg_grad_merge_ex) and the Adam sweep.  The two scratch users run one after the other on the stream and
// share one buffer.
static const int64_t DP_MAX_PAIRS = (1ll << 30) - 4096;   // == the multi-CTA gradient's limit

extern "C" int gg_dp_scratch_bytes(int32_t world, int32_t n_pairs, int32_t ld, int64_t *bytes) {
    GG_REQUIRE(bytes, "null pointer");
    GG_REQUIRE(world >= 1, "world must be >= 1");
    GG_REQUIRE(n_pairs > 0 && n_pairs <= DP_MAX_PAIRS, "n_pairs must be in 1 .. 2^30 - 4096");
    const int64_t slice = (n_pairs + (int64_t)world - 1) / world;
    int64_t grad = 0, merge = 0;
    int rc = gg_pair_grad_scratch_bytes((int32_t)slice, ld, &grad);
    if (rc) return rc;
    rc = gg_grad_merge_scratch_bytes(world, (int32_t)(2 * slice), ld, &merge);
    if (rc) return rc;
    *bytes = grad > merge ? grad : merge;
    return 0;
}

extern "C" int gg_dp_step_ex(void *comm, int32_t mode, int32_t n_pairs, const int32_t *node_id, const int32_t *node_neighbor_id,
                             const float *aux, int64_t n_node, int32_t ld, float *emb, float *m_emb, float *v_emb, float *bias,
                             float *m_bias, float *v_bias, float lambda, float *local_buf, float *gathered_buf, int32_t cap,
                             int32_t *n_unique, int32_t *uniq_ids, float *grad_rows, float *grad_bias, int32_t *row_slot,
                             float lr_t, float beta1, float beta2, float eps, void *scratch, int64_t scratch_bytes, int32_t flags,
                             void *stream) {
    GG_REQUIRE(comm, "null communicator");
    GG_REQUIRE((flags & ~GG_GRAD_MULTI_CTA) == 0, "unknown flags");
    if (n_pairs > 0 && n_pairs <= GG_MAX_BATCH && !flags)
        return gg_dp_step(comm, mode, n_pairs, node_id, node_neighbor_id, aux, n_node, ld, emb, m_emb, v_emb, bias, m_bias, v_bias,
                          lambda, local_buf, gathered_buf, cap, n_unique, uniq_ids, grad_rows, grad_bias, row_slot, lr_t, beta1,
                          beta2, eps, stream);
    gg::Comm *c = (gg::Comm *)comm;
    GG_REQUIRE(!c->p2p, "the peer-memory transport takes at most GG_MAX_BATCH pairs per step (use the NCCL transport: "
                        "gg_comm_use_p2p(comm, 0))");
    GG_REQUIRE(n_pairs > 0 && n_pairs <= DP_MAX_PAIRS, "n_pairs must be in 1 .. 2^30 - 4096");
    GG_REQUIRE(mode == 0 || mode == 1, "mode must be 0 (discriminator) or 1 (generator)");
    GG_REQUIRE(gg::ld_supported(ld), GG_LD_MESSAGE);
    GG_REQUIRE(node_id && node_neighbor_id && aux && local_buf && gathered_buf, "null pointer");
    GG_REQUIRE(cap >= 2 * (((int64_t)n_pairs + c->world - 1) / c->world), "cap too small: need 2 * ceil(n_pairs / world)");
    int lo, hi;
    block_range(n_pairs, c->rank, c->world, &lo, &hi);
    // every size check before the collective, so that a bad call fails on every rank without communicating
    int64_t need_grad = 0, need_merge = 0;
    const bool multi_grad = hi - lo > GG_MAX_BATCH || (flags & GG_GRAD_MULTI_CTA);
    if (hi > lo && multi_grad) {
        int rc = gg_pair_grad_scratch_bytes(hi - lo, ld, &need_grad);
        if (rc) return rc;
    }
    int rc = gg_grad_merge_scratch_bytes(c->world, cap, ld, &need_merge);
    if (rc) return rc;
    GG_REQUIRE(scratch && scratch_bytes >= need_grad && scratch_bytes >= need_merge,
               "scratch is null or smaller than gg_dp_scratch_bytes");
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t nf = gg_grad_buf_floats(cap, ld);
    float *rows_p = local_buf, *bias_p = local_buf + (size_t)cap * ld;
    int32_t *ids_p = (int32_t *)(bias_p + cap), *nu_p = ids_p + cap;
    if (hi > lo) {      // this rank's slice, written straight into its block; the generator loss is a mean over n_pairs
        rc = gg_pair_grad_ex(mode, hi - lo, n_pairs, node_id + lo, node_neighbor_id + lo, aux + lo, emb, bias, ld, lambda, nu_p,
                             ids_p, rows_p, bias_p, row_slot, scratch, scratch_bytes, flags, stream);
        if (rc) return rc;
    } else {
        GG_CHECK(cudaMemsetAsync(nu_p, 0, sizeof(float) * (size_t)(nf - ((size_t)cap * ld + 2 * (size_t)cap)), st));
    }
    GG_NCCL(gg::nccl().AllGather(local_buf, gathered_buf, (size_t)nf, gg::NCCL_FLOAT32, c->comm, st));   // the step's only collective
    c->collectives += 1;
    rc = gg_grad_merge_ex(c->world, cap, ld, gathered_buf, n_unique, uniq_ids, grad_rows, grad_bias, row_slot, scratch, scratch_bytes,
                          GG_GRAD_MULTI_CTA, stream);
    if (rc) return rc;
    return gg_adam_apply(n_node, ld, emb, m_emb, v_emb, bias, m_bias, v_bias, n_unique, uniq_ids, grad_rows, grad_bias, row_slot,
                         lr_t, beta1, beta2, eps, stream);
}

extern "C" int gg_dp_train_steps_ex(void *comm, int32_t mode, int64_t n_rows, const int64_t *start_list, int64_t n_starts,
                                    int32_t batch_size, const int32_t *node_id, const int32_t *node_neighbor_id, const float *aux,
                                    int64_t n_node, int32_t ld, float *emb, float *m_emb, float *v_emb, float *bias, float *m_bias,
                                    float *v_bias, float lambda, float *local_buf, float *gathered_buf, int32_t cap,
                                    int32_t *n_unique, int32_t *uniq_ids, float *grad_rows, float *grad_bias, int32_t *row_slot,
                                    float lr, float beta1, float beta2, float eps, float *beta1_power, float *beta2_power,
                                    void *scratch, int64_t scratch_bytes, int32_t flags, void *stream) {
    GG_REQUIRE(comm, "null communicator");
    GG_REQUIRE(start_list && beta1_power && beta2_power, "null host pointer");
    GG_REQUIRE((flags & ~GG_GRAD_MULTI_CTA) == 0, "unknown flags");
    GG_REQUIRE(batch_size > 0 && batch_size <= DP_MAX_PAIRS, "batch size out of range");
    if (batch_size <= GG_MAX_BATCH && !flags)
        return gg_dp_train_steps(comm, mode, n_rows, start_list, n_starts, batch_size, node_id, node_neighbor_id, aux, n_node, ld, emb,
                                 m_emb, v_emb, bias, m_bias, v_bias, lambda, local_buf, gathered_buf, cap, n_unique, uniq_ids,
                                 grad_rows, grad_bias, row_slot, lr, beta1, beta2, eps, beta1_power, beta2_power, stream);
    gg::Comm *c = (gg::Comm *)comm;
    GG_REQUIRE(!c->p2p, "the peer-memory transport takes at most GG_MAX_BATCH pairs per step (use the NCCL transport: "
                        "gg_comm_use_p2p(comm, 0))");
    GG_REQUIRE(cap >= 2 * (((int64_t)batch_size + c->world - 1) / c->world), "cap too small: need 2 * ceil(batch_size / world)");
    for (int64_t s = 0; s < n_starts; ++s) {
        const int64_t start = start_list[s];
        GG_REQUIRE(start >= 0 && start < n_rows, "start out of range");
        const int64_t end = start + batch_size < n_rows ? start + batch_size : n_rows;
        const int32_t n = (int32_t)(end - start);
        // each step lays its blocks out for its own size (a short last batch of <= GG_MAX_BATCH pairs then fits the one-CTA
        // merge); the merged result does not depend on cap
        const int32_t step_cap = (int32_t)(2 * (((int64_t)n + c->world - 1) / c->world));
        volatile float one_m_b2 = 1.0f - *beta2_power;       // lr_t as in gg_dp_train_steps
        volatile float root = sqrtf(one_m_b2);
        volatile float num = lr * root;
        volatile float den = 1.0f - *beta1_power;
        const float lr_t = num / den;
        int rc = gg_dp_step_ex(comm, mode, n, node_id + start, node_neighbor_id + start, aux + start, n_node, ld, emb, m_emb, v_emb,
                               bias, m_bias, v_bias, lambda, local_buf, gathered_buf, step_cap, n_unique, uniq_ids, grad_rows,
                               grad_bias, row_slot, lr_t, beta1, beta2, eps, scratch, scratch_bytes, flags, stream);
        if (rc) return rc;
        volatile float p1 = *beta1_power * beta1, p2 = *beta2_power * beta2;
        *beta1_power = p1;
        *beta2_power = p2;
    }
    return 0;
}
