// bfs.cu -- BFS-tree construction for a batch of roots (sm_90a).
//
// Replaces GraphGAN.construct_trees (reference src/GraphGAN/graph_gan.py:84-108).  The reference stores, per
// root, a dict node -> [father, children...]: O(N) Python objects per root and O(N^2) overall, which cannot exist
// at N >= 1e5.  Here a tree is ONE BIT PER WALK-CSR ENTRY: bit e of the root's row is set iff adj[e] is a child of
// the entry's source node in that root's tree.  The walk reads those bits next to adj[] / edge_score[] (contiguous,
// no per-neighbour probe), and the children of a node come out in adjacency order == the reference's list order
// (graph_gan.py:102-105).  The father of a node is never stored: the walk only descends, so it is the previous node.
//
// Semantics to reproduce: the father of v is the FIRST node, in the reference's FIFO order, that has v in its
// adjacency.  Since every node occurs at most once in an adjacency list of the walk CSR, "first" is decided by the
// queue position of the father alone.  Level-synchronous, one 1024-thread CTA per root, everything random lives
// in SHARED memory:
//
//   * the visited bitmap (N bits) sits in shared memory (global scratch only when N > ~1.2 M);
//   * the level's frontier is consumed in CHUNKS of consecutive queue entries holding <= 8192 adjacency entries,
//     8 consecutive entries per thread (one 32-B sector);
//   * inside a chunk, several frontier nodes may reach the same undiscovered node: every candidate entry proposes
//     key = (chunk-local index of its source, tag of the head) into a 16 k-slot shared table indexed by the head's low
//     bits, keeping the minimum (one shared-memory atomicMin per candidate entry -- a few per cent of the entries -- and
//     one barrier).  After the barrier the slot's minimum decides: same key -> this entry is THE tree edge;
//     same head, other key -> an earlier father won; other head -> hash collision, the entry stays pending and the
//     round repeats (rare: the table is at most half full).  Earlier chunks have already set their winners' visited
//     bits, so "first in queue order" holds across chunks as well;
//   * winners are compacted in entry order (a block scan) = FIFO order, appended to the queue, and their bits are
//     OR-ed into the root's tree row.
//
// The only global traffic is the adjacency stream (shared by all roots, L2), the queue (8 N bytes per root, written
// and read once, sequentially) and the tree row itself.  No per-root claim / parent / offset arrays (the round-1
// builder kept 32 N bytes of them per concurrent root and was bound by random DRAM sectors).
// HBM/L2-bound integer work; no tensor cores.
#include "gg_common.cuh"

namespace gg {
namespace {

constexpr int BFS_THREADS = 1024;
constexpr int BFS_EPT = 8;                                 // adjacency entries per thread per slab
constexpr unsigned BFS_SLAB = BFS_THREADS * BFS_EPT;       // 8192 entries
constexpr int BFS_HBITS = 14;
constexpr unsigned BFS_HSLOTS = 1u << BFS_HBITS;           // 16384 slots, 64 KB
constexpr unsigned BFS_EMPTY = 0xffffffffu;
constexpr unsigned BFS_BU_MAX = BFS_HSLOTS / 2;             // bottom-up levels sort <= 8192 64-bit keys in the table's memory
// shared memory: table | start[1025] | a0[1024] | warp totals[2][32] | pad | bitmap
constexpr unsigned BFS_FIXED_WORDS = BFS_HSLOTS + (BFS_THREADS + 1) + BFS_THREADS + 64 + 31;
constexpr long long BFS_SMEM_MAX_BYTES = 227 * 1024;
constexpr long long BFS_SMEM_BITMAP_MAX_BYTES = BFS_SMEM_MAX_BYTES - 4ll * BFS_FIXED_WORDS;

// inclusive block scan (1024 threads); `total` = sum over the block.  Two barriers; consecutive calls must alternate
// between the two halves of s_tot (a fast warp's next scan may not overwrite totals a slow warp still reads).
__device__ __forceinline__ unsigned block_scan_incl(unsigned v, unsigned *s_tot, unsigned &total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    unsigned x = v;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const unsigned y = __shfl_up_sync(FULL, x, off);
        if (lane >= off) x += y;
    }
    if (lane == 31) s_tot[wid] = x;
    __syncthreads();
    unsigned t = s_tot[lane];                               // every warp scans the 32 warp totals itself
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const unsigned y = __shfl_up_sync(FULL, t, off);
        if (lane >= off) t += y;
    }
    total = __shfl_sync(FULL, t, 31);
    const unsigned add = __shfl_sync(FULL, t, (wid + 31) & 31);
    return x + (wid ? add : 0u);
}

template <bool VSMEM>
__device__ __forceinline__ bool v_test(const unsigned *V, int w) {
    const unsigned word = VSMEM ? V[w >> 5] : __ldcg(V + (w >> 5));
    return (word >> (w & 31)) & 1u;
}

// ---------------------------------------------------------------- bottom-up level (general form)
// The top-down sweep reads every adjacency entry of the frontier and resolves "first in FIFO order" among concurrent
// proposals with the shared table.  Once the frontier's adjacency is larger than what is left undiscovered (the big
// middle levels of a small-world graph: 10-15 M frontier entries against a few M undiscovered ones), the level is
// done from the other side, with no proposal table at all:
//   phase A  every undiscovered node looks for its father = the visited neighbour with the smallest queue position
//            (all visited neighbours of an undiscovered node are on the current frontier), 8 lanes per node reading
//            whole 32-byte sectors of its adjacency, four nodes in flight per group; the winner's REVERSE entry
//            (rev[e] = index of the entry (v -> u) for e = (u -> v); static per graph, gg_reverse_entries) is the tree
//            edge: its bit is set in the root's tree row;
//   phase B  the FIFO order of the new nodes is (father's queue position, entry in the father's adjacency): the
//            frontier is re-read in queue order and each node's NEW tree bits (a node's entries carry no bits before it
//            is a father) are emitted in entry order -- the tree row doubles as the sort.  One bit per entry is read
//            where the sweep reads four bytes, a table probe and a compaction.
// Both phases stage their work lists in the (idle) proposal table.  Everything here is thread-uniform in control flow.
constexpr unsigned BU_STAGE_A = BFS_HSLOTS / 2;            // phase A: [0, 8192) node / first entry / result, [8192, 16384) end entry
constexpr unsigned BU_WIN = 2 * BFS_THREADS;               // phase B: frontier nodes per window (2 per thread)
constexpr unsigned BU_STAGE_B = BFS_HSLOTS - 2 * BU_WIN;   // phase B: [0, 12288) child entries | long list | long counts

__device__ __forceinline__ unsigned range_mask(unsigned word, unsigned wi, unsigned fw, unsigned lw, unsigned a0, unsigned a1) {
    if (wi == fw) word &= 0xffffffffu << (a0 & 31);
    if (wi == lw && (a1 & 31)) word &= (1u << (a1 & 31)) - 1u;
    return word;
}

template <bool VSMEM>
__device__ __forceinline__ void bottom_up_level(long long n_node, size_t bm_words, const unsigned *__restrict__ ip32,
                                                const int *__restrict__ adj, const int *__restrict__ rev,
                                                uint32_t *__restrict__ tb, unsigned *V, uint2 *Q, unsigned *pos,
                                                unsigned *table, unsigned *s_tot, unsigned *s_win, unsigned lo, unsigned hi,
                                                unsigned &tail, unsigned &flip, unsigned &deg_acc) {
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const unsigned nwords = (unsigned)bm_words;
    // ================= phase A: fathers
    {
        const unsigned undiscovered = (unsigned)n_node - tail;
        unsigned K = 1;                                      // bitmap words per thread per batch: ~4 k staged nodes on average
        if (undiscovered < (unsigned)(n_node >> 3)) {
            const unsigned long long k2 = ((unsigned long long)n_node >> 3) / (undiscovered ? undiscovered : 1u);
            K = k2 > 32ull ? 32u : (unsigned)k2;
            if (K < 1u) K = 1u;
        }
        const int l8 = tid & 7;
        const unsigned grp = (unsigned)tid >> 3;            // 128 groups of 8 lanes
        for (unsigned wb = 0; wb < nwords; wb += BFS_THREADS * K) {
            const unsigned w0 = wb + (unsigned)tid * K;
            unsigned cnt = 0;
            for (unsigned k = 0; k < K; ++k) {
                const unsigned wi = w0 + k;
                if (wi < nwords) {
                    unsigned word = ~(VSMEM ? V[wi] : __ldcg(V + wi));
                    if (wi == nwords - 1 && (n_node & 31)) word &= (1u << (n_node & 31)) - 1u;
                    cnt += (unsigned)__popc(word);
                }
            }
            unsigned T;
            const unsigned off = block_scan_incl(cnt, s_tot + 32 * (flip ^= 1u), T) - cnt;
            if (T == 0) continue;                           // (uniform)
            for (unsigned c0 = 0; c0 < T; c0 += BU_STAGE_A) {
                if (cnt && off < c0 + BU_STAGE_A && off + cnt > c0) {
                    unsigned idx = off;
                    for (unsigned k = 0; k < K; ++k) {
                        const unsigned wi = w0 + k;
                        if (wi >= nwords) break;
                        unsigned word = ~(VSMEM ? V[wi] : __ldcg(V + wi));
                        if (wi == nwords - 1 && (n_node & 31)) word &= (1u << (n_node & 31)) - 1u;
                        while (word) {
                            const unsigned b = (unsigned)__ffs(word) - 1u;
                            word &= word - 1u;
                            if (idx >= c0 && idx - c0 < BU_STAGE_A) table[idx - c0] = wi * 32u + b;
                            ++idx;
                        }
                    }
                }
                __syncthreads();
                const unsigned nT = (T - c0) < BU_STAGE_A ? (T - c0) : BU_STAGE_A;
                for (unsigned i = tid; i < nT; i += BFS_THREADS) {   // node -> its adjacency range (1024 independent loads)
                    const unsigned w = table[i];
                    const unsigned a0 = ip32[2 * (size_t)w], a1 = ip32[2 * (size_t)w + 2];
                    table[i] = a0; table[BU_STAGE_A + i] = a1;
                }
                __syncthreads();
                for (unsigned it = 0; it * 512u < nT; ++it) {
                    unsigned ea[4], eb[4], best[4], be[4];
#pragma unroll
                    for (int f = 0; f < 4; ++f) {
                        const unsigned i = it * 512u + (unsigned)f * 128u + grp;
                        ea[f] = 0u; eb[f] = 0u;
                        if (i < nT) { ea[f] = table[i] + (unsigned)l8; eb[f] = table[BU_STAGE_A + i]; }
                        best[f] = 0xffffffffu; be[f] = 0xffffffffu;
                    }
                    bool more = (ea[0] < eb[0]) | (ea[1] < eb[1]) | (ea[2] < eb[2]) | (ea[3] < eb[3]);
                    while (more) {
                        int u[4];
                        unsigned p[4];
#pragma unroll
                        for (int f = 0; f < 4; ++f) u[f] = (ea[f] < eb[f]) ? __ldg(adj + ea[f]) : -1;
#pragma unroll
                        for (int f = 0; f < 4; ++f) p[f] = (u[f] >= 0 && v_test<VSMEM>(V, u[f])) ? __ldcg(pos + u[f]) : 0xffffffffu;
#pragma unroll
                        for (int f = 0; f < 4; ++f) {
                            if (p[f] < best[f]) { best[f] = p[f]; be[f] = ea[f]; }
                            ea[f] += 8u;
                        }
                        more = (ea[0] < eb[0]) | (ea[1] < eb[1]) | (ea[2] < eb[2]) | (ea[3] < eb[3]);
                    }
                    __syncwarp();
#pragma unroll
                    for (int f = 0; f < 4; ++f) {
#pragma unroll
                        for (int o = 4; o >= 1; o >>= 1) {
                            const unsigned ob = __shfl_xor_sync(FULL, best[f], o), oe = __shfl_xor_sync(FULL, be[f], o);
                            if (ob < best[f]) { best[f] = ob; be[f] = oe; }
                        }
                        const unsigned i = it * 512u + (unsigned)f * 128u + grp;
                        if (l8 == 0 && i < nT) table[i] = be[f];      // this node's entry towards its father, or none
                    }
                }
                __syncthreads();
                for (unsigned i = tid; i < nT; i += BFS_THREADS) {
                    const unsigned e = table[i];
                    if (e != 0xffffffffu) {
                        const unsigned ef = (unsigned)__ldg(rev + e);    // the father's entry towards this node: the tree edge
                        atomicOr(tb + (ef >> 5), 1u << (ef & 31));
                    }
                }
                __syncthreads();
            }
        }
    }
    // ================= phase B: the new nodes in FIFO order
    {
        unsigned *stage = table, *llist = table + BU_STAGE_B, *lcnt = table + BU_STAGE_B + BU_WIN;
        for (unsigned wbase = lo; wbase < hi; wbase += BU_WIN) {
            if (tid == 0) *s_win = 0u;
            __syncthreads();
            uint2 q[2];
            unsigned cnt[2], lk[2], wd[2][3];
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                const unsigned p = wbase + 2u * (unsigned)tid + (unsigned)k;
                q[k] = (p < hi) ? Q[p] : make_uint2(0u, 0u);
                cnt[k] = 0u; lk[k] = 0xffffffffu;
                wd[k][0] = wd[k][1] = wd[k][2] = 0u;
            }
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                if (q[k].y == 0u) continue;
                const unsigned a0 = q[k].x, a1 = q[k].x + q[k].y, fw = a0 >> 5, lw = (a1 - 1u) >> 5;
                if (lw - fw < 3u) {
#pragma unroll
                    for (unsigned j = 0; j < 3; ++j)
                        if (fw + j <= lw) {
                            wd[k][j] = range_mask(__ldcg(tb + fw + j), fw + j, fw, lw, a0, a1);
                            cnt[k] += (unsigned)__popc(wd[k][j]);
                        }
                } else {                                    // more than three words of tree bits: a whole warp reads them
                    lk[k] = atomicAdd(s_win, 1u);
                    llist[lk[k]] = 2u * (unsigned)tid + (unsigned)k;
                }
            }
            __syncthreads();
            const unsigned nlong = *s_win;
            for (unsigned j = wid; j < nlong; j += 32) {
                const uint2 qq = Q[wbase + llist[j]];
                const unsigned a0 = qq.x, a1 = qq.x + qq.y, fw = a0 >> 5, lw = (a1 - 1u) >> 5;
                unsigned c = 0;
                for (unsigned wi = fw + lane; wi <= lw; wi += 32) c += (unsigned)__popc(range_mask(__ldcg(tb + wi), wi, fw, lw, a0, a1));
#pragma unroll
                for (int o = 16; o >= 1; o >>= 1) c += __shfl_xor_sync(FULL, c, o);
                if (lane == 0) lcnt[j] = c;
            }
            __syncthreads();
#pragma unroll
            for (int k = 0; k < 2; ++k) if (lk[k] != 0xffffffffu) cnt[k] = lcnt[lk[k]];
            unsigned T;
            const unsigned c2 = cnt[0] + cnt[1];
            const unsigned off = block_scan_incl(c2, s_tot + 32 * (flip ^= 1u), T) - c2;
            if (T == 0) continue;                           // (uniform) this window has no children
            // (every thread has read its long counts before the scan's barrier: the slots now carry the nodes' offsets)
            if (lk[0] != 0xffffffffu) lcnt[lk[0]] = off;
            if (lk[1] != 0xffffffffu) lcnt[lk[1]] = off + cnt[0];
            for (unsigned c0 = 0; c0 < T; c0 += BU_STAGE_B) {
                unsigned idx = off;
#pragma unroll
                for (int k = 0; k < 2; ++k) {
                    if (lk[k] == 0xffffffffu && cnt[k] && idx < c0 + BU_STAGE_B && idx + cnt[k] > c0) {
                        const unsigned fw = q[k].x >> 5;
#pragma unroll
                        for (unsigned j = 0; j < 3; ++j) {
                            unsigned word = wd[k][j];
                            while (word) {
                                const unsigned b = (unsigned)__ffs(word) - 1u;
                                word &= word - 1u;
                                if (idx >= c0 && idx - c0 < BU_STAGE_B) stage[idx - c0] = ((fw + j) << 5) + b;
                                ++idx;
                            }
                        }
                    } else {
                        idx += cnt[k];
                    }
                }
                __syncthreads();                            // (also: the long nodes' offsets are visible)
                for (unsigned j = wid; j < nlong; j += 32) {
                    unsigned run = lcnt[j];
                    if (run >= c0 + BU_STAGE_B) continue;
                    const uint2 qq = Q[wbase + llist[j]];
                    const unsigned a0 = qq.x, a1 = qq.x + qq.y, fw = a0 >> 5, lw = (a1 - 1u) >> 5;
                    for (unsigned wq = fw; wq <= lw; wq += 32) {
                        const unsigned wi = wq + lane;
                        unsigned word = (wi <= lw) ? range_mask(__ldcg(tb + wi), wi, fw, lw, a0, a1) : 0u;
                        const unsigned pc = (unsigned)__popc(word);
                        unsigned inc = pc;
#pragma unroll
                        for (int o = 1; o < 32; o <<= 1) {
                            const unsigned y = __shfl_up_sync(FULL, inc, o);
                            if (lane >= o) inc += y;
                        }
                        unsigned my = run + inc - pc;
                        while (word) {
                            const unsigned b = (unsigned)__ffs(word) - 1u;
                            word &= word - 1u;
                            if (my >= c0 && my - c0 < BU_STAGE_B) stage[my - c0] = (wi << 5) + b;
                            ++my;
                        }
                        run += __shfl_sync(FULL, inc, 31);
                        if (run >= c0 + BU_STAGE_B) break;  // (warp-uniform) the rest belongs to a later round
                    }
                }
                __syncthreads();
                const unsigned nT = (T - c0) < BU_STAGE_B ? (T - c0) : BU_STAGE_B;
                for (unsigned i = tid; i < nT; i += BFS_THREADS) {
                    const unsigned e = stage[i];
                    const int w = __ldg(adj + e);
                    const unsigned qa = ip32[2 * (size_t)w], qb = ip32[2 * (size_t)w + 2];
                    Q[tail + c0 + i] = make_uint2(qa, qb - qa);
                    pos[w] = tail + c0 + i;
                    deg_acc += qb - qa;
                    atomicOr(V + (w >> 5), 1u << (w & 31));
                }
                __syncthreads();
            }
            tail += T;
        }
        for (unsigned s = tid; s < BFS_HSLOTS; s += BFS_THREADS) table[s] = BFS_EMPTY;   // the sweep expects an empty table
    }
}

template <bool VSMEM>
__global__ void __launch_bounds__(BFS_THREADS, 1)
bfs_kernel(long long n_node, const long long *__restrict__ indptr, const int *__restrict__ adj, long long n_roots,
           const int *__restrict__ roots, uint32_t *__restrict__ tree_bits, long long tree_words, uint2 *__restrict__ qbuf,
           unsigned *__restrict__ posbuf, unsigned *__restrict__ gbitmap, int tagbits, unsigned avg_deg,
           const int *__restrict__ rev, long long nnz, float bu_ratio, int flags) {
    extern __shared__ __align__(16) unsigned bfs_smem[];
    unsigned *table = bfs_smem;
    unsigned *start = table + BFS_HSLOTS;                  // [1025] exclusive prefix of the window's degrees
    unsigned *a0s = start + BFS_THREADS + 1;               // [1024] first walk-CSR entry of the window's nodes
    unsigned *s_tot = a0s + BFS_THREADS;                   // [2][32]
    unsigned *s_win = s_tot + 64;                          // "this slab discovered something" flag
    const size_t bm_words = ((size_t)n_node + 31) / 32;
    unsigned *V = VSMEM ? (s_tot + 64 + 31) : (gbitmap + (size_t)blockIdx.x * bm_words);
    // the FIFO queue holds, per discovered node, (first walk-CSR entry, degree): all a frontier node is needed for.
    // The random indptr reads are issued when a node is APPENDED (fire and forget behind the compaction scan), so the
    // frontier sweep itself reads the queue sequentially and one window ahead.
    uint2 *Q = qbuf + (size_t)blockIdx.x * (size_t)n_node;
    unsigned *pos = posbuf + (size_t)blockIdx.x * (size_t)n_node;        // node -> queue position (bottom-up levels)
    unsigned long long *keys = reinterpret_cast<unsigned long long *>(table);   // bottom-up levels reuse the table
    const unsigned *ip32 = reinterpret_cast<const unsigned *>(indptr);   // low words (nnz < 2^31, little endian)
    const int tid = threadIdx.x;
    const unsigned tagmask = (1u << tagbits) - 1u;

    for (unsigned s = tid; s < BFS_HSLOTS; s += BFS_THREADS) table[s] = BFS_EMPTY;
    for (long long r = blockIdx.x; r < n_roots; r += gridDim.x) {
        const int root = roots[r];
        uint32_t *tb = tree_bits + (size_t)r * (size_t)tree_words;
        for (long long i = tid; i < tree_words; i += BFS_THREADS) tb[i] = 0u;
        for (size_t i = tid; i < bm_words; i += BFS_THREADS) V[i] = 0u;
        __syncthreads();
        if (tid == 0) {
            V[root >> 5] = 1u << (root & 31);
            Q[0] = make_uint2(ip32[2 * (size_t)root], ip32[2 * (size_t)root + 2] - ip32[2 * (size_t)root]);
            pos[root] = 0u;
        }
        __syncthreads();
        unsigned lo = 0, hi = 1, tail = 1, flip = 0;
        unsigned deg_acc = 0;                               // degrees of the nodes I appended during this level
        unsigned long long fe = 0;                          // adjacency entries of the current frontier (0: unknown / small)
        // adjacency entries of all discovered nodes (nnz - disc_e = entries a bottom-up level would read)
        unsigned long long disc_e = ip32[2 * (size_t)root + 2] - ip32[2 * (size_t)root];
        while (lo < hi) {                                   // one BFS level: queue entries [lo, hi)
            // ---- direction: when almost everything is discovered, the frontier's adjacency (millions of entries, hardly
            // any of them leading to a new node) is not swept; instead the few undiscovered nodes look for their father:
            // the visited neighbour with the smallest queue position (every visited neighbour of an undiscovered node is
            // on the current frontier), and the new nodes are appended sorted by (father's position, entry in the father's
            // adjacency) -- exactly the order the sweep would have produced.
            const unsigned undiscovered = (unsigned)n_node - tail;
            if (!(flags & GG_BFS_NO_SORTED_BOTTOM_UP) && undiscovered <= BFS_BU_MAX &&
                fe > 4ull * ((unsigned long long)undiscovered * avg_deg + bm_words)) {
                if (tid == 0) *s_win = 0u;
                __syncthreads();
                for (size_t wi = tid; wi < bm_words; wi += BFS_THREADS) {
                    unsigned word = ~(VSMEM ? V[wi] : __ldcg(V + wi));
                    if (wi == bm_words - 1 && (n_node & 31)) word &= (1u << (n_node & 31)) - 1u;
                    while (word) {
                        const int b = __ffs(word) - 1;
                        word &= word - 1u;
                        const int w = (int)(wi * 32 + b);
                        const unsigned a0 = ip32[2 * (size_t)w], a1 = ip32[2 * (size_t)w + 2];
                        unsigned best = 0xffffffffu;
                        for (unsigned e = a0; e < a1; ++e) {
                            const int u = __ldg(adj + e);
                            if (v_test<VSMEM>(V, u)) { const unsigned pu = __ldcg(pos + u); best = pu < best ? pu : best; }
                        }
                        if (best == 0xffffffffu) continue;   // not adjacent to the frontier (yet)
                        const uint2 fq = __ldcg(Q + best);   // the father's adjacency entries
                        unsigned ef = fq.x;
                        while (ef < fq.x + fq.y && __ldg(adj + ef) != w) ++ef;
                        keys[atomicAdd(s_win, 1u)] = ((unsigned long long)best << 32) | ef;
                    }
                }
                __syncthreads();
                const unsigned n_new = *s_win;
                unsigned n2 = 32;
                while (n2 < n_new) n2 <<= 1;
                for (unsigned i = n_new + tid; i < n2; i += BFS_THREADS) keys[i] = ~0ull;
                __syncthreads();
                for (unsigned k = 2; k <= n2; k <<= 1) {     // bitonic sort, ascending
                    for (unsigned j = k >> 1; j > 0; j >>= 1) {
                        for (unsigned i = tid; i < n2; i += BFS_THREADS) {
                            const unsigned p2 = i ^ j;
                            if (p2 > i) {
                                const unsigned long long x = keys[i], y = keys[p2];
                                if ((x > y) == ((i & k) == 0)) { keys[i] = y; keys[p2] = x; }
                            }
                        }
                        __syncthreads();
                    }
                }
                for (unsigned i = tid; i < n_new; i += BFS_THREADS) {
                    const unsigned ef = (unsigned)(keys[i] & 0xffffffffull);
                    const int w = __ldg(adj + ef);
                    const unsigned qa = ip32[2 * (size_t)w], qb = ip32[2 * (size_t)w + 2];
                    Q[tail + i] = make_uint2(qa, qb - qa);
                    pos[w] = tail + i;
                    deg_acc += qb - qa;
                    atomicOr(V + (w >> 5), 1u << (w & 31));
                    atomicOr(tb + (ef >> 5), 1u << (ef & 31));
                }
                __syncthreads();
                for (unsigned sidx = tid; sidx < 2 * BFS_BU_MAX && sidx < BFS_HSLOTS; sidx += BFS_THREADS) table[sidx] = BFS_EMPTY;
                tail += n_new;
                unsigned tot2;
                block_scan_incl(deg_acc, s_tot + 32 * (flip ^= 1u), tot2);
                fe = tot2; disc_e += tot2; deg_acc = 0;
                __syncthreads();
                lo = hi; hi = tail;
                continue;
            }
            if (rev && fe > 0 &&
                (float)((unsigned long long)nnz - disc_e) + 4.0f * (float)(hi - lo) < bu_ratio * (float)fe) {
                bottom_up_level<VSMEM>(n_node, bm_words, ip32, adj, rev, tb, V, Q, pos, table, s_tot, s_win, lo, hi, tail,
                                       flip, deg_acc);
                unsigned tot2;
                block_scan_incl(deg_acc, s_tot + 32 * (flip ^= 1u), tot2);
                fe = tot2; disc_e += tot2; deg_acc = 0;
                __syncthreads();
                lo = hi; hi = tail;
                continue;
            }
            unsigned pf_i = 0xffffffffu;                    // prefetched window (valid inside a level only)
            uint2 pf = make_uint2(0u, 0u);
            for (unsigned wbase = lo; wbase < hi; wbase += BFS_THREADS) {
                // ---- window: the next <= 1024 frontier nodes; ONE scan numbers all their adjacency entries, the
                // chunks (<= SLAB entries each) are then cut out of that numbering
                const unsigned nvalid = (hi - wbase) < (unsigned)BFS_THREADS ? (hi - wbase) : (unsigned)BFS_THREADS;
                uint2 q = make_uint2(0u, 0u);
                if (pf_i == wbase) q = pf;
                else if ((unsigned)tid < nvalid) q = Q[wbase + tid];
                pf_i = wbase + BFS_THREADS;                 // the next window of this level (written during the previous
                pf = make_uint2(0u, 0u);                    // level): in flight while this one is processed
                if (pf_i + tid < hi) pf = Q[pf_i + tid];
                unsigned tot;
                const unsigned incl = block_scan_incl(q.y, s_tot + 32 * (flip ^= 1u), tot);
                start[tid] = incl - q.y; a0s[tid] = q.x;
                if (tid == BFS_THREADS - 1) start[BFS_THREADS] = incl;
                __syncthreads();
                unsigned jlo = 0;
                while (jlo < nvalid) {                      // chunks of consecutive frontier nodes
                    const unsigned base = start[jlo];
                    unsigned m = (unsigned)__syncthreads_count((unsigned)tid >= jlo && (unsigned)tid < nvalid &&
                                                               start[tid + 1] - base <= BFS_SLAB);   // a prefix of [jlo, nvalid)
                    if (m == 0) m = 1;                      // one node with more than SLAB entries: a chunk of its own
                    if (tid == 0) *s_win = 0u;              // (the previous chunk's readers are behind the barrier above)
                    const unsigned Kend = start[jlo + m];   // entries [base, Kend) in the window's numbering
                    const bool single = (m == 1);           // a node's own entries never collide: no table needed
                    for (unsigned s0 = base; s0 < Kend; s0 += BFS_SLAB) {
                        const unsigned K0 = s0 + (unsigned)tid * BFS_EPT;
                        unsigned ee[BFS_EPT], key[BFS_EPT];
                        int w[BFS_EPT];
#pragma unroll
                        for (int x = 0; x < BFS_EPT; ++x) { ee[x] = 0xffffffffu; key[x] = 0; }
                        if (K0 < Kend) {
                            unsigned j = jlo;
                            if (!single) {                  // owner of entry K0: last j in the chunk with start[j] <= K0
                                unsigned l = jlo, h = jlo + m - 1;
                                while (l < h) {
                                    const unsigned mid = (l + h + 1) >> 1;
                                    if (start[mid] <= K0) l = mid; else h = mid - 1;
                                }
                                j = l;
                            }
                            unsigned nxt = start[j + 1];
                            if (K0 + BFS_EPT <= nxt) {      // all my entries belong to one node (the common case)
                                const unsigned e0 = a0s[j] + (K0 - start[j]);
#pragma unroll
                                for (int x = 0; x < BFS_EPT; ++x) { ee[x] = e0 + x; key[x] = (j - jlo) << tagbits; }
                            } else {
#pragma unroll
                                for (int x = 0; x < BFS_EPT; ++x) {
                                    const unsigned K = K0 + x;
                                    if (K < Kend) {
                                        while (K >= nxt) { ++j; nxt = start[j + 1]; }   // (skips empty nodes; K < Kend bounds j)
                                        ee[x] = a0s[j] + (K - start[j]);
                                        key[x] = (j - jlo) << tagbits;
                                    }
                                }
                            }
                        }
#pragma unroll
                        for (int x = 0; x < BFS_EPT; ++x) w[x] = (ee[x] != 0xffffffffu) ? __ldg(adj + ee[x]) : -1;
                        unsigned cm = 0;                    // candidate entries: head not discovered yet
#pragma unroll
                        for (int x = 0; x < BFS_EPT; ++x)
                            if (w[x] >= 0 && !v_test<VSMEM>(V, w[x])) cm |= 1u << x;
                        unsigned wm = 0;                    // winners: the tree edges among my entries
                        int anyw;
                        if (single) {
                            wm = cm;
                            if (cm) {
#pragma unroll
                                for (int x = 0; x < BFS_EPT; ++x)
                                    if ((cm >> x) & 1u) atomicOr(V + (w[x] >> 5), 1u << (w[x] & 31));
                            }
                            anyw = __syncthreads_or(wm != 0u);
                        } else {
                            unsigned pend = cm;
                            if (cm) {
#pragma unroll
                                for (int x = 0; x < BFS_EPT; ++x) key[x] |= ((unsigned)w[x] >> BFS_HBITS) & tagmask;
                            }
                            for (;;) {
                                // slot minimum: one shared-memory atomicMin per CANDIDATE entry (a few per cent of the entries) and
                                // one barrier (a barrier-per-round fixed point of plain stores was the top stall of the sweep)
                                if (pend) {
#pragma unroll
                                    for (int x = 0; x < BFS_EPT; ++x)
                                        if ((pend >> x) & 1u) atomicMin(table + ((unsigned)w[x] & (BFS_HSLOTS - 1)), key[x]);
                                }
                                __syncthreads();
                                unsigned still = 0;
                                if (pend) {
#pragma unroll
                                    for (int x = 0; x < BFS_EPT; ++x) {
                                        if (!((pend >> x) & 1u)) continue;
                                        const unsigned t = table[(unsigned)w[x] & (BFS_HSLOTS - 1)];
                                        if (t == key[x]) {
                                            wm |= 1u << x;
                                            atomicOr(V + (w[x] >> 5), 1u << (w[x] & 31));
                                        } else if ((t & tagmask) != (key[x] & tagmask)) {
                                            still |= 1u << x;   // the slot went to another head: try again
                                        }
                                    }
                                    if (wm) *s_win = 1u;
                                }
                                const int any = __syncthreads_or(still != 0u);
                                if (pend) {
#pragma unroll
                                    for (int x = 0; x < BFS_EPT; ++x)
                                        if ((pend >> x) & 1u) table[(unsigned)w[x] & (BFS_HSLOTS - 1)] = BFS_EMPTY;
                                }
                                pend = still;
                                if (!any) break;
                                __syncthreads();
                            }
                            anyw = (int)*s_win;
                        }
                        if (!anyw) continue;                // (uniform) nothing discovered by this slab: no compaction
                        // ---- winners in entry order = FIFO order.  They are sparse (a few per cent of the entries), so
                        // they are first compacted into the (now idle, all-EMPTY) table as (head, entry) pairs at their FIFO
                        // index, then handled one per thread: entry range of the node -> queue, queue position, tree bit.
                        unsigned ntot;
                        const unsigned cnt = (unsigned)__popc(wm);
                        unsigned li = block_scan_incl(cnt, s_tot + 32 * (flip ^= 1u), ntot) - cnt;
                        if (wm) {
#pragma unroll
                            for (int x = 0; x < BFS_EPT; ++x) {
                                if (!((wm >> x) & 1u)) continue;
                                table[2 * li] = (unsigned)w[x];
                                table[2 * li + 1] = ee[x];
                                ++li;
                            }
                        }
                        __syncthreads();
                        for (unsigned i = tid; i < ntot; i += BFS_THREADS) {
                            const unsigned wv = table[2 * i], e = table[2 * i + 1];
                            table[2 * i] = BFS_EMPTY; table[2 * i + 1] = BFS_EMPTY;
                            const unsigned qa = ip32[2 * (size_t)wv], qb = ip32[2 * (size_t)wv + 2];
                            Q[tail + i] = make_uint2(qa, qb - qa);
                            pos[wv] = tail + i;
                            deg_acc += qb - qa;
                            atomicOr(tb + (e >> 5), 1u << (e & 31));
                        }
                        tail += ntot;
                        // the table reads / resets above must be over before the next slab's atomicMin proposals (a late
                        // reset would wipe a proposal)
                        if (!single || s0 + BFS_SLAB < Kend) __syncthreads();
                    }
                    jlo += m;
                }
            }
            {                                               // adjacency entries of the next frontier
                unsigned tot2;
                block_scan_incl(deg_acc, s_tot + 32 * (flip ^= 1u), tot2);
                fe = tot2; disc_e += tot2; deg_acc = 0;
            }
            __syncthreads();                                // the queue entries appended above are read next
            lo = hi; hi = tail;
        }
    }
}

// tree row -> parent array (tests / compatibility): parent[adj[e]] = source(e) for every set bit e
__global__ void tree_parent_kernel(long long n_node, const long long *__restrict__ indptr, const int *__restrict__ adj,
                                   long long n_roots, const uint32_t *__restrict__ tree_bits, long long tree_words,
                                   int *__restrict__ parent) {
    const long long r = blockIdx.y;
    const uint32_t *tb = tree_bits + (size_t)r * (size_t)tree_words;
    int *par = parent + (size_t)r * (size_t)n_node;
    for (long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x; u < n_node; u += (long long)gridDim.x * blockDim.x) {
        const long long a0 = indptr[u], a1 = indptr[u + 1];
        for (long long e = a0; e < a1; ++e)
            if ((tb[e >> 5] >> (e & 31)) & 1u) par[adj[e]] = (int)u;
    }
}

// rev[e] for e = (u -> v): the index of the entry (v -> u).  One warp per source node, 8 lanes per entry scanning the
// head's adjacency a 32-byte sector at a time.  Entries without a reverse (an asymmetric CSR) get -1 and are counted.
__global__ void reverse_entries_kernel(long long n_node, const long long *__restrict__ indptr, const int *__restrict__ adj,
                                       int *__restrict__ rev, int *__restrict__ n_missing) {
    const int lane = threadIdx.x & 31, l8 = lane & 7, g = lane >> 3;
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long u = warp; u < n_node; u += nwarps) {
        const long long a0 = indptr[u], a1 = indptr[u + 1];
        for (long long e0 = a0; e0 < a1; e0 += 4) {          // (warp-uniform trip count: the shuffles below need every lane)
            const long long e = e0 + g;
            int found = -1;
            if (e < a1) {
                const int v = __ldg(adj + e);
                const long long b0 = indptr[v], b1 = indptr[v + 1];
                for (long long x = b0 + l8; x < b1 && found < 0; x += 8)
                    if (__ldg(adj + x) == (int)u) found = (int)x;
            }
            __syncwarp();
#pragma unroll
            for (int o = 4; o >= 1; o >>= 1) {
                const int other = __shfl_xor_sync(FULL, found, o);
                found = other > found ? other : found;
            }
            if (l8 == 0 && e < a1) {
                rev[e] = found;
                if (found < 0) atomicAdd(n_missing, 1);
            }
        }
    }
}

constexpr float BFS_BU_RATIO_DEFAULT = 1.0f;   // bottom-up when (undiscovered entries + 4 * frontier nodes) < ratio * frontier entries

int bfs_tagbits(long long n_node) {
    int bits = 0;
    while (bits < 40 && (1ll << bits) < n_node) ++bits;     // ids < 2^bits
    return bits > BFS_HBITS ? bits - BFS_HBITS : 0;
}

}  // namespace
}  // namespace gg

extern "C" int gg_tree_words(int64_t nnz, int64_t *words) {
    GG_REQUIRE(words && nnz >= 0, "bad arguments");
    *words = (nnz + 31) / 32 + 1;
    return 0;
}

extern "C" int gg_bfs_scratch_bytes(int64_t n_node, int64_t nnz, int64_t *bytes) {
    GG_REQUIRE(bytes && n_node >= 0 && nnz >= 0, "bad arguments");
    const long long bm_bytes = (n_node + 31) / 32 * 4;
    const bool in_smem = bm_bytes <= gg::BFS_SMEM_BITMAP_MAX_BYTES;
    *bytes = (int64_t)gg::sm_count() * (12 * n_node + (in_smem ? 0 : bm_bytes)) + 16;
    return 0;
}

extern "C" int gg_reverse_entries(int64_t n_node, int64_t nnz, const int64_t *indptr, const int32_t *adj, int32_t *rev,
                                  int32_t *n_missing, void *stream) {
    GG_REQUIRE(indptr && adj && rev && n_missing, "null pointer");
    GG_REQUIRE(nnz < 0x7ffffff0ll, "too many adjacency entries for 32-bit entry numbers");
    cudaStream_t st = (cudaStream_t)stream;
    GG_CHECK(cudaMemsetAsync(n_missing, 0, sizeof(int32_t), st));
    if (n_node == 0 || nnz == 0) return 0;
    long long blocks = (n_node * 32 + 255) / 256;
    const long long cap = (long long)gg::sm_count() * 32;
    if (blocks > cap) blocks = cap;
    gg::reverse_entries_kernel<<<(unsigned)blocks, 256, 0, st>>>(n_node, (const long long *)indptr, adj, rev, n_missing);
    return gg::check_cuda(cudaGetLastError(), "reverse entries kernel launch");
}

extern "C" int gg_bfs_build_ex(int64_t n_node, int64_t nnz, const int64_t *indptr, const int32_t *adj, const int32_t *rev,
                               int64_t n_roots, const int32_t *roots, uint32_t *tree_bits, int64_t tree_words,
                               void *scratch, int64_t scratch_bytes, float bottom_up_ratio, int32_t flags, void *stream) {
    GG_REQUIRE(indptr && adj && roots && tree_bits && scratch, "null pointer");
    GG_REQUIRE(nnz < 0x7ffffff0ll, "too many adjacency entries for 32-bit entry numbers");
    GG_REQUIRE(tree_words >= (nnz + 31) / 32, "tree_words too small (gg_tree_words)");
    GG_REQUIRE(flags >= 0 && flags <= GG_BFS_NO_SORTED_BOTTOM_UP, "unknown flags");
    if (n_roots == 0 || n_node == 0) return 0;
    const long long bm_bytes = (n_node + 31) / 32 * 4;
    const bool in_smem = bm_bytes <= gg::BFS_SMEM_BITMAP_MAX_BYTES;
    const int64_t per_cta = 12 * n_node + (in_smem ? 0 : bm_bytes);
    int64_t ctas = scratch_bytes / per_cta;
    if (ctas > gg::sm_count()) ctas = gg::sm_count();
    if (ctas > n_roots) ctas = n_roots;
    GG_REQUIRE(ctas >= 1, "scratch too small");
    const int tagbits = gg::bfs_tagbits(n_node);
    GG_REQUIRE(tagbits + 10 <= 31, "graph too large for the 32-bit proposal keys");
    uint2 *qbuf = (uint2 *)scratch;
    unsigned *posbuf = (unsigned *)(qbuf + (size_t)ctas * (size_t)n_node);
    unsigned *gbm = in_smem ? nullptr : posbuf + (size_t)ctas * (size_t)n_node;
    const unsigned avg_deg = (unsigned)((nnz + n_node - 1) / n_node > 0 ? (nnz + n_node - 1) / n_node : 1);
    const size_t smem = 4 * (size_t)gg::BFS_FIXED_WORDS + (in_smem ? (size_t)bm_bytes : 0);
    const float ratio = bottom_up_ratio < 0.0f ? gg::BFS_BU_RATIO_DEFAULT : bottom_up_ratio;
    cudaStream_t st = (cudaStream_t)stream;
    if (in_smem) {
        GG_CHECK(cudaFuncSetAttribute(gg::bfs_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        gg::bfs_kernel<true><<<(unsigned)ctas, gg::BFS_THREADS, smem, st>>>(
            n_node, (const long long *)indptr, adj, n_roots, roots, tree_bits, tree_words, qbuf, posbuf, gbm, tagbits, avg_deg,
            rev, nnz, ratio, flags);
    } else {
        GG_CHECK(cudaFuncSetAttribute(gg::bfs_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        gg::bfs_kernel<false><<<(unsigned)ctas, gg::BFS_THREADS, smem, st>>>(
            n_node, (const long long *)indptr, adj, n_roots, roots, tree_bits, tree_words, qbuf, posbuf, gbm, tagbits, avg_deg,
            rev, nnz, ratio, flags);
    }
    return gg::check_cuda(cudaGetLastError(), "bfs kernel launch");
}

extern "C" int gg_bfs_build(int64_t n_node, int64_t nnz, const int64_t *indptr, const int32_t *adj, int64_t n_roots,
                            const int32_t *roots, uint32_t *tree_bits, int64_t tree_words, void *scratch,
                            int64_t scratch_bytes, void *stream) {
    return gg_bfs_build_ex(n_node, nnz, indptr, adj, nullptr, n_roots, roots, tree_bits, tree_words, scratch, scratch_bytes,
                           -1.0f, 0, stream);
}

extern "C" int gg_tree_parent(int64_t n_node, const int64_t *indptr, const int32_t *adj, int64_t n_roots,
                              const int32_t *roots, const uint32_t *tree_bits, int64_t tree_words, int32_t *parent,
                              void *stream) {
    GG_REQUIRE(indptr && adj && tree_bits && parent, "null pointer");
    (void)roots;
    if (n_roots == 0 || n_node == 0) return 0;
    GG_REQUIRE(n_roots <= 65535, "at most 65535 roots per call");
    cudaStream_t st = (cudaStream_t)stream;
    GG_CHECK(cudaMemsetAsync(parent, 0xff, sizeof(int32_t) * (size_t)n_roots * (size_t)n_node, st));
    long long bx = (n_node + 255) / 256;
    if (bx > 4096) bx = 4096;
    gg::tree_parent_kernel<<<dim3((unsigned)bx, (unsigned)n_roots), 256, 0, st>>>(
        n_node, (const long long *)indptr, adj, n_roots, tree_bits, tree_words, parent);
    return gg::check_cuda(cudaGetLastError(), "tree parent kernel launch");
}
