// grad_multi.cu -- K2 for mini-batches of any size: the sparse gradient of pair_grad_body computed by the whole grid.
//
// Same outputs, bit for bit, as the one-CTA pair_grad_kernel (update_dev.cuh) on every batch it accepts, and for larger
// batches the same sequential IndexedSlices sum (TF1.8 unique + segment_sum) it restates:
//   entries   t = 0..E-1 (E = 2B): the i-side of pairs 0..B-1, then the j-side;  id(t) = node_id[t] or node_neighbor_id[t-B]
//   slots     unique rows numbered in order of first occurrence;  uniq_ids[slot] = id,  row_slot[id] = slot
//   rows      grad_rows[slot][c] = +0 (+) term(t)[c] over the slot's entries in entry order, one __fadd_rn chain per
//             coordinate;  term = __fadd_rn(__fmul_rn(d, other row), __fmul_rn(lambda, own row))
//   bias      grad_bias[slot] = the same chain over the j-side entries: d + lambda * bias (D) or d (G)
// Stages (all on the caller's stream, scratch from gg_pair_grad_scratch_bytes, nothing allocated):
//   1 forward     grid-stride 8-lane groups: delta[B] (pair_delta, shared with the one-CTA kernel);  every entry does an
//                 unsigned atomicMin of t on row_slot[id] (all -1 = UINT_MAX on entry) -> first entry of every row
//   2 slots       first-occurrence flags counted per tile, tile offsets by launch_exclusive_scan_i64, then numbered
//   3 grouping    stable LSD radix sort (8-bit digits) of the entry indices by slot -> entries grouped by slot, entry
//                 order inside a slot
//   4 terms       each entry's term vector (and bias term, +0 for i-side entries) written in grouped order
//   5 sums        slots of <= SHORT_MAX entries: one 8-lane group each (as pair_sums);  longer slots: one CTA each, one
//                 thread per column, the slot's contiguous terms streamed through a cp.async ring in shared memory so
//                 that ~200 KB of loads are in flight while the adds run in entry order
// A slot's chain is serial by contract, so the longest slot bounds the last stage (DESIGN.md section 5, K2).
//
// gg_grad_merge_ex (data-parallel merge of `world` compact gradients, any size) reuses stages 2 and 3 on the entries of
// the gathered blocks (number_and_group over MergeEntries): the ids are read and their row_slot cleared in one launch,
// first entries found by atomicMin in the next, and the sums read the rows in place through the sorted entry index.
#include "update_dev.cuh"

namespace gg {
namespace {

constexpr int MC_THREADS = 1024;       // entries per tile of the slot numbering / threads of the radix kernels
constexpr int RADIX_ITEMS = 4;         // entries per thread of a radix tile
constexpr int RADIX_TILE = MC_THREADS * RADIX_ITEMS;
constexpr int SHORT_MAX = 16;          // longest slot summed by an 8-lane group
constexpr int LONG_THREADS = 512;
constexpr int LONG_STAGES = 6;         // cp.async ring: LONG_STAGES x LONG_STAGE_FLOATS floats of shared memory
constexpr int LONG_STAGE_FLOATS = 8192;
constexpr long long MAX_PAIRS = (1ll << 30) - 4096;   // E = 2B and every entry index (rounded up to a tile) fit in int32

__host__ __device__ inline int term_stride(int ld) { return ld + 4; }   // row terms, bias term, 3 floats of padding

struct Scratch {
    float *delta;              // [B]
    long long *tile_cnt;       // [n_tiles + 1] first occurrences per numbering tile -> exclusive offsets
    int *key[2], *val[2];      // [E] radix ping-pong: slot and entry index
    long long *hist;           // [256 * radix tiles + 1]
    int *off;                  // [E + 1] slot -> first grouped position
    int *long_list;            // [E / (SHORT_MAX + 1) + 1]
    int *counters;             // [0] long slots listed, [1] long slots taken
    float *terms;              // [E, term_stride(ld)]
    size_t bytes;
};

inline size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }

Scratch carve(char *base, long long B, int ld) {
    const long long E = 2 * B;
    const long long n_tiles = (E + MC_THREADS - 1) / MC_THREADS, r_tiles = (E + RADIX_TILE - 1) / RADIX_TILE;
    Scratch s;
    size_t at = 0;
    auto take = [&](size_t bytes) { char *p = base ? base + at : nullptr; at += align_up(bytes); return p; };
    s.delta = (float *)take(4 * B);
    s.tile_cnt = (long long *)take(8 * (n_tiles + 1));
    for (int k = 0; k < 2; ++k) { s.key[k] = (int *)take(4 * E); s.val[k] = (int *)take(4 * E); }
    s.hist = (long long *)take(8 * (256 * r_tiles + 1));
    s.off = (int *)take(4 * (E + 1));
    s.long_list = (int *)take(4 * (E / (SHORT_MAX + 1) + 1));
    s.counters = (int *)take(4 * 2);
    s.terms = (float *)take(4 * (size_t)E * term_stride(ld));
    s.bytes = at;
    return s;
}

__device__ __forceinline__ int entry_id(int t, int B, const int *ni, const int *nj) { return t < B ? ni[t] : nj[t - B]; }

// ---- 1: forward pass + first entry of every row
__global__ void __launch_bounds__(256) mc_forward_kernel(int mode, int B, int batch_total, const int *__restrict__ ni,
                                                         const int *__restrict__ nj, const float *__restrict__ aux,
                                                         const float *__restrict__ emb, const float *__restrict__ bias,
                                                         int ld, float *__restrict__ delta, int *row_slot) {
    const int lane = threadIdx.x & 31, grp = lane >> 3, g = lane & 7;
    const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, nthr = (long long)gridDim.x * blockDim.x;
    for (long long k0 = (tid >> 5) * 4; k0 < B; k0 += (nthr >> 5) * 4) {
        const int k = (int)k0 + grp;
        const bool valid = k < B;
        const int i = valid ? ni[k] : 0, j = valid ? nj[k] : 0;
        const float a_k = valid ? aux[k] : 0.0f;
        const float d = pair_delta<false>(mode, batch_total, i, j, a_k, emb, bias, ld, g);
        if (valid && g == 0) delta[k] = d;
    }
    for (long long t = tid; t < 2ll * B; t += nthr)
        atomicMin(reinterpret_cast<unsigned *>(row_slot) + entry_id((int)t, B, ni, nj), (unsigned)t);
}

// ---- 2: slots.  row_slot[id] holds the row's first entry (stage 1) until that entry overwrites it with the slot,
// which is never larger; so an entry reads "first" exactly when row_slot[id] == t, whichever value it sees.
__device__ __forceinline__ int block_excl_scan(int x) {   // MC_THREADS threads
    __shared__ int s_warp[32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int v = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(FULL, v, o);
        if (lane >= o) v += y;
    }
    if (lane == 31) s_warp[wid] = v;
    __syncthreads();
    if (wid == 0) {
        int w = s_warp[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(FULL, w, o);
            if (lane >= o) w += y;
        }
        s_warp[lane] = w;
    }
    __syncthreads();
    const int excl = (wid ? s_warp[wid - 1] : 0) + v - x;
    __syncthreads();
    return excl;
}

// Where the grouping stages (2, 3) read entry t's row id: the pair entries of a mini-batch, or the slots of the
// gathered blocks of gg_grad_merge_ex (id -1: rank r has no slot s).  An absent entry is never a first occurrence and
// sorts after every slot (key E).
struct PairEntries {
    int B;
    const int *ni, *nj;
    __device__ __forceinline__ int id(int t) const { return entry_id(t, B, ni, nj); }
};
struct MergeEntries {
    const int *ids;
    __device__ __forceinline__ int id(int t) const { return ids[t]; }
};

template <class Src>
__global__ void __launch_bounds__(MC_THREADS) mc_count_kernel(int E, Src src, const int *row_slot, long long *__restrict__ tile_cnt) {
    const int t = blockIdx.x * MC_THREADS + threadIdx.x;
    const int id = t < E ? src.id(t) : -1;
    const int first = (id >= 0 && row_slot[id] == t) ? 1 : 0;
    const int n = __syncthreads_count(first);
    if (threadIdx.x == 0) tile_cnt[blockIdx.x] = n;
}

template <class Src>
__global__ void __launch_bounds__(MC_THREADS) mc_number_kernel(int E, Src src, const long long *__restrict__ tile_off, int n_tiles,
                                                               int *row_slot, int *__restrict__ uniq_ids, int *__restrict__ n_unique) {
    const int t = blockIdx.x * MC_THREADS + threadIdx.x;
    const int id = t < E ? src.id(t) : -1;
    const int first = (id >= 0 && row_slot[id] == t) ? 1 : 0;
    const int excl = block_excl_scan(first);
    if (first) {
        const int slot = (int)tile_off[blockIdx.x] + excl;
        uniq_ids[slot] = id;
        row_slot[id] = slot;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) *n_unique = (int)tile_off[n_tiles];
}

// ---- 3: stable LSD radix sort of (slot, entry) by slot
template <class Src>
__global__ void __launch_bounds__(MC_THREADS) mc_keys_kernel(int E, Src src, const int *__restrict__ row_slot, int *__restrict__ key,
                                                             int *__restrict__ val) {
    const long long t = (long long)blockIdx.x * MC_THREADS + threadIdx.x;
    if (t < E) {
        const int id = src.id((int)t);
        key[t] = id >= 0 ? row_slot[id] : E;
        val[t] = (int)t;
    }
}

__global__ void __launch_bounds__(MC_THREADS) mc_hist_kernel(int E, const int *__restrict__ key, int shift, int r_tiles,
                                                             long long *__restrict__ hist) {
    __shared__ int cnt[256];
    if (threadIdx.x < 256) cnt[threadIdx.x] = 0;
    __syncthreads();
    const long long base = (long long)blockIdx.x * RADIX_TILE;
#pragma unroll
    for (int r = 0; r < RADIX_ITEMS; ++r) {
        const long long q = base + r * MC_THREADS + threadIdx.x;
        if (q < E) atomicAdd(&cnt[(key[q] >> shift) & 255], 1);
    }
    __syncthreads();
    if (threadIdx.x < 256) hist[(long long)threadIdx.x * r_tiles + blockIdx.x] = cnt[threadIdx.x];
}

// Entries keep their order inside a digit: in round r the tile's entries r*1024 .. r*1024+1023 are ranked by warp
// (match + lanes below) and across warps (per-digit prefix over the 32 warps), on top of the earlier rounds' counts.
__global__ void __launch_bounds__(MC_THREADS) mc_scatter_kernel(int E, const int *__restrict__ key_in, const int *__restrict__ val_in,
                                                                int shift, int r_tiles, const long long *__restrict__ hist,
                                                                int *__restrict__ key_out, int *__restrict__ val_out) {
    __shared__ int wcnt[32 * 256];
    __shared__ int dbase[256];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid < 256) dbase[tid] = 0;
    const unsigned lt = (1u << lane) - 1u;
    const long long base = (long long)blockIdx.x * RADIX_TILE;
    for (int r = 0; r < RADIX_ITEMS; ++r) {
        const long long q = base + r * MC_THREADS + tid;
        const bool valid = q < E;
        const int k = valid ? key_in[q] : 0, v = valid ? val_in[q] : 0;
        const int dg = valid ? (k >> shift) & 255 : 256;
        for (int x = tid; x < 32 * 256; x += MC_THREADS) wcnt[x] = 0;
        __syncthreads();
        const unsigned peers = __match_any_sync(FULL, dg);
        const int wr = __popc(peers & lt);
        if (valid && wr == 0) wcnt[wid * 256 + dg] = __popc(peers);
        __syncthreads();
        if (tid < 256) {
            int s = dbase[tid];
            for (int w = 0; w < 32; ++w) { const int c = wcnt[w * 256 + tid]; wcnt[w * 256 + tid] = s; s += c; }
            dbase[tid] = s;
        }
        __syncthreads();
        if (valid) {
            const long long dst = hist[(long long)dg * r_tiles + blockIdx.x] + wcnt[wid * 256 + dg] + wr;
            key_out[dst] = k;
            val_out[dst] = v;
        }
        __syncthreads();
    }
}

// ---- 4: slot offsets and the term vectors, in grouped order (one 8-lane group per entry)
__global__ void __launch_bounds__(256) mc_terms_kernel(int mode, int B, const int *__restrict__ ni, const int *__restrict__ nj,
                                                       const float *__restrict__ emb, const float *__restrict__ bias, int ld,
                                                       float lambda, const float *__restrict__ delta, const int *__restrict__ key,
                                                       const int *__restrict__ val, int *__restrict__ off, float *__restrict__ terms) {
    const int lane = threadIdx.x & 31, g = lane & 7;
    const long long gid = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
    const long long ngrp = ((long long)gridDim.x * blockDim.x) >> 3;
    const int E = 2 * B, ts = term_stride(ld);
    for (long long p = gid; p < E; p += ngrp) {
        const int t = val[p], u = key[p];
        if (g == 0 && (p == 0 || key[p - 1] != u)) off[u] = (int)p;
        if (g == 0 && p == E - 1) off[u + 1] = E;
        const int side = t < B ? t : t - B;
        const int self = t < B ? ni[side] : nj[side], other = t < B ? nj[side] : ni[side];
        const float d = delta[side];
        const float *srow = emb + (size_t)self * ld, *orow = emb + (size_t)other * ld;
        float *out = terms + (size_t)p * ts;
        for (int c = 4 * g; c < ld; c += 32) {
            const float4 o = ldg4(orow + c), s = ldg4(srow + c);
            float4 v;
            v.x = __fadd_rn(__fmul_rn(d, o.x), __fmul_rn(lambda, s.x));
            v.y = __fadd_rn(__fmul_rn(d, o.y), __fmul_rn(lambda, s.y));
            v.z = __fadd_rn(__fmul_rn(d, o.z), __fmul_rn(lambda, s.z));
            v.w = __fadd_rn(__fmul_rn(d, o.w), __fmul_rn(lambda, s.w));
            *reinterpret_cast<float4 *>(out + c) = v;
        }
        // bias: j-side entries only (generator.py:28-29 has no bias l2).  An i-side entry adds +0, which leaves the
        // chain's bits unchanged: a sum that starts at +0 is never -0.
        if (g == 0) {
            float b = 0.0f;
            if (t >= B) b = mode == 0 ? __fadd_rn(d, __fmul_rn(lambda, __ldg(bias + self))) : d;
            *reinterpret_cast<float4 *>(out + ld) = make_float4(b, 0.f, 0.f, 0.f);
        }
    }
}

// ---- 5a: short slots, 8 lanes each (columns in passes of 64, four entries' terms in flight); longer slots are listed
__global__ void __launch_bounds__(256) mc_short_sums_kernel(int E, int ld, const int *__restrict__ n_unique,
                                                            const int *__restrict__ off, const float *__restrict__ terms,
                                                            float *__restrict__ grad_rows, float *__restrict__ grad_bias,
                                                            int *__restrict__ long_list, int *__restrict__ counters) {
    const int g = threadIdx.x & 7;
    const long long gid = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
    const long long ngrp = ((long long)gridDim.x * blockDim.x) >> 3;
    const int U = *n_unique, ts = term_stride(ld);
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long long u = gid; u < U; u += ngrp) {
        const int lo = off[u], n = off[u + 1] - lo;
        if (n > SHORT_MAX) {
            if (g == 0) long_list[atomicAdd(&counters[0], 1)] = (int)u;
            continue;
        }
        const float *base = terms + (size_t)lo * ts;
        for (int c0 = 0; c0 < ld; c0 += 64) {
            const int c = c0 + 4 * g;
            const bool two = c + 32 < ld;
            float4 acc0 = z, acc1 = z;
            for (int r = 0; r < n; r += 4) {
                float4 o0[4], o1[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const bool in = r + e < n;
                    const float *tp = base + (size_t)(r + e) * ts + c;
                    o0[e] = in ? ldg4(tp) : z;
                    o1[e] = (in && two) ? ldg4(tp + 32) : z;
                }
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    if (r + e >= n) break;
                    acc0.x = __fadd_rn(acc0.x, o0[e].x); acc0.y = __fadd_rn(acc0.y, o0[e].y);
                    acc0.z = __fadd_rn(acc0.z, o0[e].z); acc0.w = __fadd_rn(acc0.w, o0[e].w);
                    acc1.x = __fadd_rn(acc1.x, o1[e].x); acc1.y = __fadd_rn(acc1.y, o1[e].y);
                    acc1.z = __fadd_rn(acc1.z, o1[e].z); acc1.w = __fadd_rn(acc1.w, o1[e].w);
                }
            }
            *reinterpret_cast<float4 *>(grad_rows + (size_t)u * ld + c) = acc0;
            if (two) *reinterpret_cast<float4 *>(grad_rows + (size_t)u * ld + c + 32) = acc1;
        }
        if (g == 0) {
            float gb = 0.0f;
            for (int r = 0; r < n; ++r) gb = __fadd_rn(gb, __ldg(base + (size_t)r * ts + ld));
            grad_bias[u] = gb;
        }
    }
}

// ---- 5b: long slots, one CTA each (taken from the list in any order), thread c < ld sums column c, thread ld the bias (at
// ld = LONG_THREADS there is no such thread: mc_long_bias_kernel sums it)
__device__ __forceinline__ void cp_async16(void *dst, const void *src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_ring() { asm volatile("cp.async.wait_group %0;" ::"n"(LONG_STAGES - 1) : "memory"); }

__global__ void __launch_bounds__(LONG_THREADS, 1) mc_long_sums_kernel(int ld, const int *__restrict__ off, const float *__restrict__ terms,
                                                                       float *__restrict__ grad_rows, float *__restrict__ grad_bias,
                                                                       const int *__restrict__ long_list, int *counters) {
    extern __shared__ float4 ring4[];
    float *ring = reinterpret_cast<float *>(ring4);
    __shared__ int s_u;
    const int tid = threadIdx.x, ts = term_stride(ld);
    const int se = LONG_STAGE_FLOATS / ts;             // entries per stage
    for (;;) {
        if (tid == 0) {
            const int k = atomicAdd(&counters[1], 1);
            s_u = k < *(volatile int *)&counters[0] ? long_list[k] : -1;
        }
        __syncthreads();
        const int u = s_u;
        if (u < 0) break;
        const int lo = off[u], n = off[u + 1] - lo;
        const float *src = terms + (size_t)lo * ts;
        const int n_st = (n + se - 1) / se;
        auto issue = [&](int s) {
            if (s < n_st) {
                const int e0 = s * se, ne = min(se, n - e0);
                const float *g = src + (size_t)e0 * ts;
                float *dst = ring + (s % LONG_STAGES) * LONG_STAGE_FLOATS;
                for (int k = tid; k < ne * ts / 4; k += LONG_THREADS) cp_async16(dst + 4 * k, g + 4 * k);
            }
            cp_async_commit();
        };
        for (int s = 0; s < LONG_STAGES - 1; ++s) issue(s);
        float acc = 0.0f;
        for (int s = 0; s < n_st; ++s) {
            issue(s + LONG_STAGES - 1);                  // into the stage consumed in the previous iteration
            cp_async_wait_ring();
            __syncthreads();
            if (tid <= ld) {
                const float *b = ring + (s % LONG_STAGES) * LONG_STAGE_FLOATS + tid;
                const int ne = min(se, n - s * se);
#pragma unroll 8
                for (int e = 0; e < ne; ++e) acc = __fadd_rn(acc, b[e * ts]);
            }
            __syncthreads();
        }
        if (tid < ld) grad_rows[(size_t)u * ld + tid] = acc;
        else if (tid == ld) grad_bias[u] = acc;
    }
}

// ---- 5c (ld >= LONG_THREADS only): the bias of the long slots, which mc_long_sums_kernel has no thread left for.  One
// warp per slot: every lane loads one entry's bias term per group of 32 entries, LONG_BIAS_TILES groups at a time (the
// next LONG_BIAS_TILES groups' loads in flight while these are added), and the warp adds them in entry order through
// shuffles -- the same +0-started __fadd_rn chain that thread `ld` would run, at one dependent add per entry.
constexpr int LONG_BIAS_TILES = 8;
__global__ void __launch_bounds__(256) mc_long_bias_kernel(int ld, const int *__restrict__ off, const float *__restrict__ terms,
                                                           float *__restrict__ grad_bias, const int *__restrict__ long_list,
                                                           const int *__restrict__ counters) {
    constexpr int U = LONG_BIAS_TILES;
    const int lane = threadIdx.x & 31;
    const int warp = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), nwarps = (int)((gridDim.x * blockDim.x) >> 5);
    const int ts = term_stride(ld), n_long = counters[0];
    for (int k = warp; k < n_long; k += nwarps) {
        const int u = long_list[k], lo = off[u], n = off[u + 1] - lo;
        const float *b = terms + (size_t)lo * ts + ld;
        float acc = 0.0f, nxt[U];
#pragma unroll
        for (int q = 0; q < U; ++q) nxt[q] = (32 * q + lane < n) ? __ldg(b + (size_t)(32 * q + lane) * ts) : 0.0f;
        for (int e0 = 0; e0 < n; e0 += 32 * U) {
            float cur[U];
#pragma unroll
            for (int q = 0; q < U; ++q) {
                cur[q] = nxt[q];
                const int e = e0 + 32 * (U + q) + lane;
                nxt[q] = (e < n) ? __ldg(b + (size_t)e * ts) : 0.0f;
            }
#pragma unroll
            for (int q = 0; q < U; ++q) {
                const int left = n - (e0 + 32 * q);        // warp-uniform
                if (left >= 32) {
#pragma unroll
                    for (int t = 0; t < 32; ++t) acc = __fadd_rn(acc, __shfl_sync(FULL, cur[q], t));
                } else {
                    for (int t = 0; t < left; ++t) acc = __fadd_rn(acc, __shfl_sync(FULL, cur[q], t));
                }
            }
        }
        if (lane == 0) grad_bias[u] = acc;
    }
}

// Stages 2 + 3 on the caller's stream for E entries whose ids `src` gives, with row_slot[id] = first entry of the row:
// slots, uniq_ids, n_unique, then the entries (val) sorted by slot (key; absent entries, key E, last).  keys <= max_key.
// *cur: the ping-pong half that holds the sorted arrays.
template <class Src>
int number_and_group(const Src &src, int E, int max_key, int *row_slot, int *uniq_ids, int *n_unique, long long *tile_cnt,
                     long long *hist, int *const key[2], int *const val[2], cudaStream_t st, int *cur) {
    const int n_tiles = (E + MC_THREADS - 1) / MC_THREADS, r_tiles = (E + RADIX_TILE - 1) / RADIX_TILE;
    mc_count_kernel<<<n_tiles, MC_THREADS, 0, st>>>(E, src, row_slot, tile_cnt);
    GG_CHECK(cudaGetLastError());
    int rc = launch_exclusive_scan_i64(tile_cnt, n_tiles, nullptr, st);
    if (rc) return rc;
    mc_number_kernel<<<n_tiles, MC_THREADS, 0, st>>>(E, src, tile_cnt, n_tiles, row_slot, uniq_ids, n_unique);
    GG_CHECK(cudaGetLastError());
    mc_keys_kernel<<<n_tiles, MC_THREADS, 0, st>>>(E, src, row_slot, key[0], val[0]);
    GG_CHECK(cudaGetLastError());
    int bits = 1;
    while (bits < 31 && (max_key >> bits) != 0) ++bits;
    int c = 0;
    for (int shift = 0; shift < bits; shift += 8, c ^= 1) {
        mc_hist_kernel<<<r_tiles, MC_THREADS, 0, st>>>(E, key[c], shift, r_tiles, hist);
        GG_CHECK(cudaGetLastError());
        rc = launch_exclusive_scan_i64(hist, 256ll * r_tiles, nullptr, st);
        if (rc) return rc;
        mc_scatter_kernel<<<r_tiles, MC_THREADS, 0, st>>>(E, key[c], val[c], shift, r_tiles, hist, key[c ^ 1], val[c ^ 1]);
        GG_CHECK(cudaGetLastError());
    }
    *cur = c;
    return 0;
}

// ---------------------------------------------------------------- multi-CTA data-parallel merge (gg_grad_merge_ex)
// The contract of grad_merge_body (update_dev.cuh) for any number of entries: entry t = r * cap + s for s < nu_r, slots
// in first-occurrence order over t, per slot one +0-started __fadd_rn chain over its entries in increasing t (= rank
// order).  A rank's block holds every id once, so a slot has at most `world` entries: one 8-lane group per slot sums
// it, reading the rows in the gathered buffer through the sorted entry index (no term copy, no long-slot path).
struct MergeScratch {
    int *ids;                  // [E] entry -> row id, -1 where s >= nu_r
    long long *tile_cnt;       // [n_tiles + 1]
    int *key[2], *val[2];      // [E] radix ping-pong: slot (E = absent) and entry index
    long long *hist;           // [256 * radix tiles + 1]
    int *off;                  // [E + 1] slot -> first grouped position
    size_t bytes;
};

MergeScratch carve_merge(char *base, long long E) {
    const long long n_tiles = (E + MC_THREADS - 1) / MC_THREADS, r_tiles = (E + RADIX_TILE - 1) / RADIX_TILE;
    MergeScratch s;
    size_t at = 0;
    auto take = [&](size_t bytes) { char *p = base ? base + at : nullptr; at += align_up(bytes); return p; };
    s.ids = (int *)take(4 * E);
    s.tile_cnt = (long long *)take(8 * (n_tiles + 1));
    for (int k = 0; k < 2; ++k) { s.key[k] = (int *)take(4 * E); s.val[k] = (int *)take(4 * E); }
    s.hist = (long long *)take(8 * (256 * r_tiles + 1));
    s.off = (int *)take(4 * (E + 1));
    s.bytes = at;
    return s;
}

__host__ __device__ inline size_t merge_stride(int cap, int ld) { return (size_t)cap * ld + 2 * (size_t)cap + 4; }   // == gg_grad_buf_floats

// ---- merge 1: every entry's id, and row_slot[id] = -1 for every id present (it may still hold this rank's local slots
// from the slice gradient).  A launch of its own: the first-occurrence atomicMin below must see all of them cleared.
__global__ void __launch_bounds__(256) mg_ids_kernel(int E, int cap, int ld, const float *__restrict__ gathered, int *__restrict__ ids,
                                                     int *row_slot) {
    const size_t stride = merge_stride(cap, ld);
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < E; t += (long long)gridDim.x * blockDim.x) {
        const int r = (int)(t / cap), s = (int)(t - (long long)r * cap);
        const float *tail = gathered + (size_t)r * stride + (size_t)cap * ld;       // bias | ids | n_unique
        const int nu = __float_as_int(__ldg(tail + 2 * (size_t)cap));
        const int id = s < nu ? __float_as_int(__ldg(tail + cap + s)) : -1;
        ids[t] = id;
        if (id >= 0) row_slot[id] = -1;
    }
}

// ---- merge 2: first entry of every row (row_slot = -1 = UINT_MAX everywhere it is read)
__global__ void __launch_bounds__(256) mg_first_kernel(int E, const int *__restrict__ ids, int *row_slot) {
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < E; t += (long long)gridDim.x * blockDim.x) {
        const int id = ids[t];
        if (id >= 0) atomicMin(reinterpret_cast<unsigned *>(row_slot) + id, (unsigned)t);
    }
}

// ---- merge 3: slot -> [off[u], off[u + 1]) in grouped order (both ends written; neighbours write equal values)
__global__ void __launch_bounds__(256) mg_offsets_kernel(int E, const int *__restrict__ key, int *__restrict__ off) {
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < E; p += (long long)gridDim.x * blockDim.x) {
        const int u = key[p];
        if (u == E) continue;
        if (p == 0 || key[p - 1] != u) off[u] = (int)p;
        if (p == E - 1 || key[p + 1] != u) off[u + 1] = (int)p + 1;
    }
}

// ---- merge 4: sums, one 8-lane group per slot (columns in passes of 64, four entries' rows in flight), entries in t order
__global__ void __launch_bounds__(256) mg_sums_kernel(int cap, int ld, const float *__restrict__ gathered, const int *__restrict__ n_unique,
                                                      const int *__restrict__ off, const int *__restrict__ val,
                                                      float *__restrict__ grad_rows, float *__restrict__ grad_bias) {
    const int g = threadIdx.x & 7;
    const long long gid = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
    const long long ngrp = ((long long)gridDim.x * blockDim.x) >> 3;
    const int U = *n_unique;
    const size_t stride = merge_stride(cap, ld);
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    auto row_of = [&](int t) {        // rows[s] of rank r's block
        const int r = t / cap;
        return gathered + (size_t)r * stride + (size_t)(t - r * cap) * ld;
    };
    for (long long u = gid; u < U; u += ngrp) {
        const int lo = off[u], n = off[u + 1] - lo;
        for (int c0 = 0; c0 < ld; c0 += 64) {
            const int c = c0 + 4 * g;
            const bool two = c + 32 < ld;
            float4 acc0 = z, acc1 = z;
            for (int r = 0; r < n; r += 4) {
                float4 o0[4], o1[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const bool in = r + e < n;
                    const float *tp = row_of(in ? val[lo + r + e] : 0) + c;
                    o0[e] = in ? ldg4(tp) : z;
                    o1[e] = (in && two) ? ldg4(tp + 32) : z;
                }
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    if (r + e >= n) break;
                    acc0.x = __fadd_rn(acc0.x, o0[e].x); acc0.y = __fadd_rn(acc0.y, o0[e].y);
                    acc0.z = __fadd_rn(acc0.z, o0[e].z); acc0.w = __fadd_rn(acc0.w, o0[e].w);
                    acc1.x = __fadd_rn(acc1.x, o1[e].x); acc1.y = __fadd_rn(acc1.y, o1[e].y);
                    acc1.z = __fadd_rn(acc1.z, o1[e].z); acc1.w = __fadd_rn(acc1.w, o1[e].w);
                }
            }
            *reinterpret_cast<float4 *>(grad_rows + (size_t)u * ld + c) = acc0;
            if (two) *reinterpret_cast<float4 *>(grad_rows + (size_t)u * ld + c + 32) = acc1;
        }
        if (g == 0) {
            float gb = 0.0f;
            for (int r = 0; r < n; ++r) {
                const int t = val[lo + r], k = t / cap;
                gb = __fadd_rn(gb, __ldg(gathered + (size_t)k * stride + (size_t)cap * ld + (t - k * cap)));
            }
            grad_bias[u] = gb;
        }
    }
}

}  // namespace
}  // namespace gg

extern "C" int gg_pair_grad_scratch_bytes(int32_t n_pairs, int32_t ld, int64_t *bytes) {
    GG_REQUIRE(bytes, "null pointer");
    GG_REQUIRE(n_pairs > 0 && n_pairs <= gg::MAX_PAIRS, "n_pairs must be in 1 .. 2^30 - 4096");
    GG_REQUIRE(gg::ld_supported(ld), GG_LD_MESSAGE);
    *bytes = (int64_t)gg::carve(nullptr, n_pairs, ld).bytes;
    return 0;
}

extern "C" int gg_pair_grad_ex(int32_t mode, int32_t n_pairs, int32_t batch_total, const int32_t *node_id,
                               const int32_t *node_neighbor_id, const float *aux, const float *emb, const float *bias, int32_t ld,
                               float lambda, int32_t *n_unique, int32_t *uniq_ids, float *grad_rows, float *grad_bias,
                               int32_t *row_slot, void *scratch, int64_t scratch_bytes, int32_t flags, void *stream) {
    GG_REQUIRE(mode == 0 || mode == 1, "mode must be 0 (discriminator) or 1 (generator)");
    GG_REQUIRE(n_pairs > 0 && n_pairs <= gg::MAX_PAIRS, "n_pairs must be in 1 .. 2^30 - 4096");
    GG_REQUIRE((flags & ~GG_GRAD_MULTI_CTA) == 0, "unknown flags");
    if (n_pairs <= GG_MAX_BATCH && !(flags & GG_GRAD_MULTI_CTA))
        return gg_pair_grad(mode, n_pairs, batch_total, node_id, node_neighbor_id, aux, emb, bias, ld, lambda, n_unique,
                            uniq_ids, grad_rows, grad_bias, row_slot, stream);
    GG_REQUIRE(node_id && node_neighbor_id && aux && emb && bias && n_unique && uniq_ids && grad_rows && grad_bias && row_slot,
               "null pointer");
    GG_REQUIRE(gg::ld_supported(ld), GG_LD_MESSAGE);
    const gg::Scratch need = gg::carve(nullptr, n_pairs, ld);
    GG_REQUIRE(scratch && scratch_bytes >= (int64_t)need.bytes, "scratch is null or smaller than gg_pair_grad_scratch_bytes");
    GG_REQUIRE(((uintptr_t)scratch & 255) == 0, "scratch must be 256-byte aligned");
    const gg::Scratch s = gg::carve((char *)scratch, n_pairs, ld);
    cudaStream_t st = (cudaStream_t)stream;
    const int B = n_pairs, E = 2 * n_pairs;
    const int grid = gg::sm_count() * 8;
    gg::mc_forward_kernel<<<grid, 256, 0, st>>>(mode, B, batch_total > 0 ? batch_total : B, node_id, node_neighbor_id, aux, emb,
                                                 bias, ld, s.delta, row_slot);
    GG_CHECK(cudaGetLastError());
    int cur = 0;                                    // slots are < E
    int rc = gg::number_and_group(gg::PairEntries{B, node_id, node_neighbor_id}, E, E - 1, row_slot, uniq_ids, n_unique, s.tile_cnt,
                                  s.hist, s.key, s.val, st, &cur);
    if (rc) return rc;
    gg::mc_terms_kernel<<<grid, 256, 0, st>>>(mode, B, node_id, node_neighbor_id, emb, bias, ld, lambda, s.delta, s.key[cur],
                                               s.val[cur], s.off, s.terms);
    GG_CHECK(cudaGetLastError());
    GG_CHECK(cudaMemsetAsync(s.counters, 0, 2 * sizeof(int), st));
    gg::mc_short_sums_kernel<<<grid, 256, 0, st>>>(E, ld, n_unique, s.off, s.terms, grad_rows, grad_bias, s.long_list, s.counters);
    GG_CHECK(cudaGetLastError());
    const size_t smem = sizeof(float) * gg::LONG_STAGES * gg::LONG_STAGE_FLOATS;
    GG_CHECK(cudaFuncSetAttribute(gg::mc_long_sums_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int long_grid = E / (gg::SHORT_MAX + 1);
    if (long_grid > gg::sm_count()) long_grid = gg::sm_count();
    if (long_grid > 0) {
        gg::mc_long_sums_kernel<<<long_grid, gg::LONG_THREADS, smem, st>>>(ld, s.off, s.terms, grad_rows, grad_bias, s.long_list,
                                                                            s.counters);
        GG_CHECK(cudaGetLastError());
        if (ld >= gg::LONG_THREADS) {
            int bias_blocks = (E / (gg::SHORT_MAX + 1) + 7) / 8;     // a warp per possible long slot, 8 per CTA
            if (bias_blocks > gg::sm_count() * 8) bias_blocks = gg::sm_count() * 8;
            gg::mc_long_bias_kernel<<<bias_blocks, 256, 0, st>>>(ld, s.off, s.terms, grad_bias, s.long_list, s.counters);
            GG_CHECK(cudaGetLastError());
        }
    }
    return 0;
}

extern "C" int gg_grad_merge_scratch_bytes(int32_t world, int32_t cap, int32_t ld, int64_t *bytes) {
    GG_REQUIRE(bytes, "null pointer");
    GG_REQUIRE(world >= 1 && cap >= 1, "world and cap must be >= 1");
    GG_REQUIRE((int64_t)world * cap <= 2 * gg::MAX_PAIRS, "world * cap must be at most 2^31 - 8192 entries");
    GG_REQUIRE(gg::ld_supported(ld), GG_LD_MESSAGE);
    *bytes = (int64_t)gg::carve_merge(nullptr, (long long)world * cap).bytes;
    return 0;
}

extern "C" int gg_grad_merge_ex(int32_t world, int32_t cap, int32_t ld, const float *gathered, int32_t *n_unique,
                                int32_t *uniq_ids, float *grad_rows, float *grad_bias, int32_t *row_slot, void *scratch,
                                int64_t scratch_bytes, int32_t flags, void *stream) {
    GG_REQUIRE((flags & ~GG_GRAD_MULTI_CTA) == 0, "unknown flags");
    GG_REQUIRE(world >= 1 && cap >= 1, "world and cap must be >= 1");
    GG_REQUIRE((int64_t)world * cap <= 2 * gg::MAX_PAIRS, "world * cap must be at most 2^31 - 8192 entries");
    if ((int64_t)world * cap <= 2 * GG_MAX_BATCH * 8 && !(flags & GG_GRAD_MULTI_CTA))
        return gg_grad_merge(world, cap, ld, gathered, n_unique, uniq_ids, grad_rows, grad_bias, row_slot, stream);
    GG_REQUIRE(gathered && n_unique && uniq_ids && grad_rows && grad_bias && row_slot, "null pointer");
    GG_REQUIRE(gg::ld_supported(ld), GG_LD_MESSAGE);
    GG_REQUIRE(world == 1 || cap % 2 == 0, "cap must be even when world > 1 (16-byte aligned blocks)");
    GG_REQUIRE(((uintptr_t)gathered & 15) == 0, "gathered must be 16-byte aligned");
    const int E = world * cap;
    const gg::MergeScratch need = gg::carve_merge(nullptr, E);
    GG_REQUIRE(scratch && scratch_bytes >= (int64_t)need.bytes, "scratch is null or smaller than gg_grad_merge_scratch_bytes");
    GG_REQUIRE(((uintptr_t)scratch & 255) == 0, "scratch must be 256-byte aligned");
    const gg::MergeScratch s = gg::carve_merge((char *)scratch, E);
    cudaStream_t st = (cudaStream_t)stream;
    const int grid = gg::sm_count() * 8;
    gg::mg_ids_kernel<<<grid, 256, 0, st>>>(E, cap, ld, gathered, s.ids, row_slot);
    GG_CHECK(cudaGetLastError());
    gg::mg_first_kernel<<<grid, 256, 0, st>>>(E, s.ids, row_slot);
    GG_CHECK(cudaGetLastError());
    int cur = 0;                                    // slots are < E, absent entries have key E
    int rc = gg::number_and_group(gg::MergeEntries{s.ids}, E, E, row_slot, uniq_ids, n_unique, s.tile_cnt, s.hist, s.key, s.val, st,
                                  &cur);
    if (rc) return rc;
    gg::mg_offsets_kernel<<<grid, 256, 0, st>>>(E, s.key[cur], s.off);
    GG_CHECK(cudaGetLastError());
    gg::mg_sums_kernel<<<grid, 256, 0, st>>>(cap, ld, gathered, n_unique, s.off, s.val[cur], grad_rows, grad_bias);
    return gg::check_cuda(cudaGetLastError(), "merge sums launch");
}
