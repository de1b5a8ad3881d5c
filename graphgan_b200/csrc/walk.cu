// walk.cu -- K1, the graph-softmax walk sampler (sm_90a).
//
// Replaces GraphGAN.sample (reference src/GraphGAN/graph_gan.py:225-270) for a whole batch of
// roots: one warp owns one walk at a time (persistent CTAs pull walk ids from a global
// counter).  Per step the warp
//   1. enumerates the candidate list [father] + children(cur) from the walk CSR and the
//      root's BFS parent array (children = adjacency entries whose father is cur, in
//      adjacency order == the reference's list order, graph_gan.py:96,102-105);
//   2. scores the candidates on demand: generator.all_score[cur, cand] = e_cur . e_cand + b_cand
//      (generator.py:21) -- four 8-lane groups, each streaming one embedding row per
//      LDG.128 quartet (one full 128 B line per group per instruction);
//   3. softmax (utils.py:131-133) + float64 CDF + inverse-CDF draw (numpy legacy
//      RandomState.choice, called at graph_gan.py:262) with warp shuffles.
// The arithmetic is the canonical sequence of DESIGN.md section 3 == oracle/gg_oracle.c.
#include <string.h>

#include "walk_list.cuh"

namespace gg {
namespace {

struct Rng {
    int mode;
    uint32_t k0, k1, tag;
    const double *stream;
    long long n_stream;
    long long cursor;  // GG_RNG_STREAM only
    int exhausted;
    __device__ __forceinline__ double draw(uint32_t root, uint32_t walk, uint32_t step) {
        if (mode == GG_RNG_PHILOX) {
            uint32_t a, b;
            philox4x32_10(root, walk, step, tag, k0, k1, a, b);
            return u53(a, b);
        }
        if (cursor >= n_stream) { exhausted = 1; return 0.0; }
        return stream[cursor++];
    }
};

// One complete walk, executed by a full warp.  Returns the status.
// a (root, depth-1 child) pair gets a shared CDF (step1_cdf_kernel) when at least this many walks picked it
#ifndef GG_S1_MIN_WALKS
#define GG_S1_MIN_WALKS 1
#endif
constexpr int S1_MIN_WALKS = GG_S1_MIN_WALKS;

// Does the pair (root slot, i-th neighbour) at `s1pos` get a shared CDF from step1_cdf_kernel?  With S1_MIN_WALKS = 1: every
// pair that was picked (measured: hub lists are long and the builder's queue starts the longest first; 2 -- pairs picked
// once stay inside their walk -- and "2, or 1 when the child is score-cached" were both slower with the flat steps).
__device__ __forceinline__ bool s1_is_shared(const gg_walk_desc &d, long long s1pos) {
    return __ldg(d.s1_cnt + s1pos) >= S1_MIN_WALKS;
}

// where a walk (re)starts: a fresh walk stands on its root; a walk handed over by the level-synchronous steps
// (flat_*_kernel below) continues from the node it reached (step == choices made so far)
struct WalkState {
    int cur, prev, step, fedge, suml;
};

template <int CPL>
__device__ __forceinline__ int walk_one(const gg_walk_desc &d, Rng &rng, int slot, uint32_t k, long long w,
                                        int *s_ids, float *s_sc, int *g_ids, float *g_sc, int lane,
                                        unsigned long long &raw_steps, unsigned long long &raw_suml,
                                        unsigned long long &overflow, unsigned long long &rows_gathered,
                                        unsigned int (&cyc)[7], Stage &stg, const WalkState *from = nullptr) {
    const int root = d.roots[slot];
    const uint32_t *tb = d.tree_bits + (size_t)slot * (size_t)d.tree_words;
    int cur = root, prev = -1, step = 0, fedge = -1, plen = 0;
    int steps = 0, suml = 0, status = GG_NOTRUN, sample = -1;
    int32_t *prow = (d.max_path > 0 && d.paths) ? d.paths + (size_t)w * (size_t)d.max_path : nullptr;
    if (from) {
        cur = from->cur; prev = from->prev; step = from->step; fedge = from->fedge; steps = from->step; suml = from->suml;
        plen = step + 1;
    } else {
        if (prow && lane == 0) prow[0] = cur;
        plen = 1;
    }
    const int steps_in = steps, suml_in = suml;

    const long long t_walk = clock64();
    for (;;) {
        const long long t_step = clock64();
        const long long a0 = d.indptr[cur], a1 = d.indptr[cur + 1];
        int n, idx, nxt;
        bool inc_father = false;
        long long s1pos = -1;     // slice of the depth-1 cache, when this (root, child) pair was picked by >= 2 walks
        if (step == 1 && d.s1_q) {
            s1pos = __ldg(d.rq_ptr + slot) + (fedge - d.indptr[root]);
            if (!s1_is_shared(d, s1pos)) s1pos = -1;
        }
        if (step == 0 && d.root_q) {
            // ---- root step from the per-root CDF (hub.cu: root_cdf_kernel): every walk of a root
            // sees the same candidate list tree[root][1:] and the same scores, so the softmax/CDF
            // is computed once per root per pass and each walk only inverts it.
            n = (int)(a1 - a0);
            if (n == 0) { status = GG_VOID; break; }  // graph_gan.py:252-253
            const double u = rng.draw((uint32_t)root, k, 0u);
            if (rng.exhausted) { status = GG_NOTRUN; break; }
            idx = d.first_idx ? __ldg(d.first_idx + w) : cdf_search(d.root_q + __ldg(d.rq_ptr + slot), n, u);
            nxt = __ldg(d.adj + a0 + idx);
        } else if (s1pos >= 0) {
            // ---- depth-1 step from the per-(root, child) CDF (step1_cdf_kernel): walks of a root that picked the
            // same child share one candidate list; it was built once, each walk only inverts it
            n = __ldg(d.s1_n + s1pos);
            if (n == 0) { status = GG_VOID; break; }  // graph_gan.py:255-257
            inc_father = !d.for_d && !((d.d1_bits[fedge >> 5] >> (fedge & 31)) & 1u);
            const double u = rng.draw((uint32_t)root, k, 1u);
            const long long o = __ldg(d.s1_ptr + s1pos);
            idx = (n == 1) ? 0 : cdf_search_raw(d.s1_q + o, n, u);
            nxt = __ldg(d.s1_ids + o + idx);
        } else {
            // ---- candidate list (graph_gan.py:250-259) + scores
            inc_father = step > 0;
            if (d.for_d && step == 1) inc_father = false;
            if (!d.for_d && step == 1 && ((d.d1_bits[fedge >> 5] >> (fedge & 31)) & 1u)) inc_father = false;
            int *ids; float *sc; float m;
            build_list<CPL, UNR>(d, tb, cur, prev, inc_father, s_ids, s_sc, g_ids, g_sc, lane, n, m, ids, sc, rows_gathered, cyc, stg);
            if (n == 0) { status = GG_VOID; break; }  // graph_gan.py:252-257

            // ---- softmax + inverse CDF (utils.py:131-133, np.random.choice at graph_gan.py:262)
            const long long t_c = clock64();
            const double u = rng.draw((uint32_t)root, k, (uint32_t)step);   // the stream mode consumes it regardless
            if (rng.exhausted) { status = GG_NOTRUN; break; }
            idx = (n == 1) ? 0 : choose_index(sc, n, m, u, lane, sc != s_sc ? reinterpret_cast<double *>(s_sc) : nullptr);
            nxt = ids[idx];
            __syncwarp();
            cyc[2] += (unsigned int)(clock64() - t_c);
        }
        cyc[step == 0 ? 3 : (step == 1 ? 4 : 5)] += (unsigned int)(clock64() - t_step);   // (dynamic index: keeps the counters in local memory, off the register budget)
        if (step == 0) fedge = (int)(a0 + idx);  // every walk-CSR neighbour of the root is its child
        if (prow && lane == 0 && plen < d.max_path) prow[plen] = nxt;
        ++plen;
        ++steps; suml += n;
        if (inc_father && idx == 0) { sample = cur; status = GG_DONE; break; }  // graph_gan.py:264-266
        prev = cur; cur = nxt; ++step;
    }
    cyc[6] += (unsigned int)(clock64() - t_walk);
    raw_steps += (unsigned)(steps - steps_in); raw_suml += (unsigned)(suml - suml_in);
    if (lane == 0) {
        d.samples[w] = sample;
        d.status[w] = status;
        d.first_edge[w] = fedge;
        d.wsteps[w] = steps;
        d.wsuml[w] = suml;
        if (d.path_len) d.path_len[w] = (status == GG_DONE) ? plen : 0;
    }
    if (status == GG_DONE && d.max_path > 0 && plen > d.max_path) overflow += 1;
    return status;
}

// ---------------------------------------------------------------- depth-1 reuse (Philox mode)
// root_step_kernel: the root step of every walk (one thread per walk inverts the root's CDF) and a count of
// the walks per (root, depth-1 child).  step1_cdf_kernel: for every pair picked by >= S1_MIN_WALKS walks, the
// child's candidate list / softmax / un-normalised CDF + total, built ONCE (walk_kernel then inverts it per walk;
// a pair picked once is cheaper inside its walk, which needs no CDF array).
__global__ void root_step_kernel(const __grid_constant__ gg_walk_desc d) {
    const long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= d.n_walks) return;
    const int slot = __ldg(d.walk_slot + w);
    const int root = d.roots[slot];
    const uint32_t k = (uint32_t)(w - __ldg(d.walk_ptr + slot));
    const uint32_t k0 = (uint32_t)d.seed, k1 = (uint32_t)(d.seed >> 32);
    uint32_t a, b;
    if (d.update_ratio < 1.0) {
        philox4x32_10((uint32_t)root, 0xffffffffu, 0u, d.pass_tag, k0, k1, a, b);
        if (!(u53(a, b) < d.update_ratio)) { d.first_idx[w] = -2; return; }
    }
    const long long a0 = d.indptr[root];
    const int n = (int)(d.indptr[root + 1] - a0);
    if (n == 0) { d.first_idx[w] = -1; return; }
    philox4x32_10((uint32_t)root, k, 0u, d.pass_tag, k0, k1, a, b);
    const long long o = __ldg(d.rq_ptr + slot);
    const int idx = cdf_search(d.root_q + o, n, u53(a, b));
    d.first_idx[w] = idx;
    atomicAdd(d.s1_cnt + o + idx, 1);
}

// Queue items that are one pair each.  The queue is sorted by decreasing child degree, and a chunk of S1_CHUNK pairs runs
// on one warp, so the pairs must be short by the time chunks start: at C3 the 8192nd pair's child still has ~3 000
// neighbours (a chunk there is ~16 such lists in series: the launch's tail), the 65 536th ~140.  Measured at C3 on the
// H100: 8192 -> 1.01 ms for the depth-1 stage, 32768 and 65536 -> 0.83 ms (DESIGN.md section 8.1).
#ifndef GG_S1_SINGLES
#define GG_S1_SINGLES 65536
#endif
constexpr int S1_SINGLES = GG_S1_SINGLES, S1_CHUNK = 16;

template <int CPL>
__global__ void __launch_bounds__(WARPS_PER_CTA * 32, walk_min_ctas(CPL)) step1_cdf_kernel(const __grid_constant__ gg_walk_desc d) {
    extern __shared__ __align__(16) unsigned char walk_smem[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    float *s_sc = reinterpret_cast<float *>(walk_smem + (size_t)wid * WALK_SMEM_PER_WARP);
    int *s_ids = reinterpret_cast<int *>(s_sc + SC_CAP);
    Stage stg;
    stg.buf = s_sc;
    stg.bar = reinterpret_cast<unsigned long long *>(s_ids + ID_CAP);
    stg.phase = 0u;
    stg.on = !d.no_tma && d.edge_score != nullptr;
    if (stg.on) {
        if (lane == 0) {
            mbar_init(stg.bar, 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncwarp();
    }
    const long long gw = (long long)blockIdx.x * WARPS_PER_CTA + wid;
    const long long nwarps = (long long)gridDim.x * WARPS_PER_CTA;
    int *g_ids = reinterpret_cast<int *>(d.scratch) + (size_t)gw * 2 * (size_t)d.max_cand;
    float *g_sc = reinterpret_cast<float *>(g_ids + d.max_cand);
    unsigned long long rows_gathered = 0;
    unsigned int cyc[7] = {0, 0, 0, 0, 0, 0, 0};
    // queue mode (s1_order): the first S1_SINGLES items are single pairs (the largest lists, one warp each, started
    // first); after them one item is a chunk of S1_CHUNK pairs (most pairs were never picked: one atomic per
    // chunk keeps the queue cheap).  Without s1_order: static striding.
    long long item = gw, sub = 0, sub_end = 0;
    const long long n_single = d.s1_nq < S1_SINGLES ? d.s1_nq : S1_SINGLES;
    const long long n_items = n_single + (d.s1_nq - n_single + S1_CHUNK - 1) / S1_CHUNK;
    for (;;) {
        long long pos;
        if (d.s1_order) {
            if (sub >= sub_end) {
                unsigned int it = 0;
                if (lane == 0) it = atomicAdd(d.work_counter, 1u);
                it = __shfl_sync(FULL, it, 0);
                if ((long long)it >= n_items) break;
                if ((long long)it < n_single) { sub = it; sub_end = sub + 1; }
                else { sub = n_single + ((long long)it - n_single) * S1_CHUNK; sub_end = sub + S1_CHUNK < d.s1_nq ? sub + S1_CHUNK : d.s1_nq; }
            }
            pos = __ldg(d.s1_order + sub);
            ++sub;
        } else {
            if (item >= d.s1_nq) break;
            pos = item;
            item += nwarps;
        }
        if (!s1_is_shared(d, pos)) continue;
        const int slot = __ldg(d.s1_slot + pos);
        const int root = d.roots[slot];
        const uint32_t *tb = d.tree_bits + (size_t)slot * (size_t)d.tree_words;
        const long long e = d.indptr[root] + (pos - __ldg(d.rq_ptr + slot));
        const int c = __ldg(d.adj + e);
        const bool inc_father = !d.for_d && !((d.d1_bits[e >> 5] >> (e & 31)) & 1u);   // graph_gan.py:258-259
        int n; float m; int *ids; float *sc;
        // a list too long for the warp's shared id buffer is enumerated straight into its slice of the pool (degree + 1
        // entries): no copy from the global scratch afterwards
        build_list<CPL, UNR_S1>(d, tb, c, root, inc_father, s_ids, s_sc, d.s1_ids + __ldg(d.s1_ptr + pos), g_sc, lane, n, m, ids, sc,
                                rows_gathered, cyc, stg);
        if (lane == 0) d.s1_n[pos] = n;
        if (n == 0) continue;
        const long long o = __ldg(d.s1_ptr + pos);
        if (ids == s_ids)
            for (int i = lane; i < n; i += 32) d.s1_ids[o + i] = ids[i];
        if (n > 1) cdf_store_raw<UNR_S1>(sc, n, m, d.s1_q + o, lane);
        __syncwarp();
    }
    if (lane == 0 && rows_gathered) atomicAdd(d.counters + GG_CNT_ROWS_GATHERED, rows_gathered);
}

// ---------------------------------------------------------------- order-free (Philox) kernel
// FlatView: the buffers of the level-synchronous steps (see below), carved out of gg_walk_desc.flat_buf.
struct FlatView {
    int4 *list[2];         // [W] walks that execute step s next, as records (walk, node it stands on, node it came from,
                           //     root slot): list[s & 1] -- one 16-byte load gives a kernel everything about the walk
    int4 *tail;            // [W] walks the persistent kernel finishes (after the last level-synchronous step), same records
    int *hub;              // [W] per level: items (indices into the level's list) that stand on a score-cached node; on a
                           //     level that groups them (SHARE_HUB): the records that own a distinct hub key
    int *item_n;           // [W] per item: candidate-list length | father flag << 30 (0: nothing left to do for the item)
    int *pool_ids;         // [W * stride] per item: its candidate ids
    unsigned *ctr;         // counters: [0] tail length; level s: [1 + 4 s + {0: items, 1: hub items, 2: distinct keys of a
                           //     shared level that are not score-cached, 3: work queue}]; after them, level s of a level that
                           //     groups hub items: [FLAT_CTR_WORDS + 3 s + {0: hub owners, 1: hub work items, 2: members placed}]
    int stride;            // pool entries per item (>= hub_threshold: a node below the threshold has fewer neighbours)
    int steps;             // level-synchronous steps 1 .. steps
    // shared levels (SHARE_LEVELS): one candidate list + CDF per distinct (root slot, node), every walk on it draws from it
    unsigned long long *keys;   // [tbl_mask + 1] open-addressing table of slot * n_node + node (empty: ~0)
    int *owner;            // [tbl_mask + 1] per table slot: the record that inserted the key (its item owns the list)
    int *rec_slot;         // [W] per record: its table slot (-1: a hub item, run per walk; -2 - slot: a grouped hub item)
    int *uniq;             // [W] the level's distinct keys that are not score-cached, as the records that own them
    double *pool_cdf;      // [W * (stride + 1)] per owning item: its un-normalised CDF and the total (cdf_store_raw)
    unsigned long long tbl_mask;
    // hub groups (SHARE_HUB): the walks of a shared level on one score-cached (root slot, node) are drawn by one warp
    unsigned *gcnt;        // [tbl_mask + 1] per table slot: walks on the hub key
    unsigned *gpos;        // [tbl_mask + 1] per table slot: the next free place of the key's range of hub_rec
    int *hub_rec;          // [W] the hub records, each group contiguous
    int4 *hub_work;        // [W] work items: (owner record, first place in hub_rec, members, 0), <= HUB_GROUP_MAX members
};
constexpr int FLAT_MAX_STEPS = 14;
constexpr int FLAT_CTR_WORDS = 1 + 4 * (FLAT_MAX_STEPS + 2);
constexpr int FLAT_CTR_ALL = FLAT_CTR_WORDS + 3 * (FLAT_MAX_STEPS + 2);
#define GG_FCTR(fv, s, k) ((fv).ctr + 1 + 4 * (s) + (k))
#define GG_FCTR_HUB(fv, s, k) ((fv).ctr + FLAT_CTR_WORDS + 3 * (s) + (k))
// the record list of level s (a select: a run-time index into the kernel parameter would copy it to local memory)
__device__ __forceinline__ int4 *level_list(const FlatView &fv, int s) { return (s & 1) ? fv.list[1] : fv.list[0]; }

// Levels whose walks share one candidate list per distinct (root slot, node): bit s = level s, s >= 2 only (from step 2 on
// the list is [tree father] + children(node) and depends on nothing else of the walk; step 1 is the depth-1 reuse).
// 0 = no sharing: every level runs flat_enum + flat_choose per walk.
#ifndef GG_SHARE_LEVELS
#define GG_SHARE_LEVELS 0x4
#endif
constexpr unsigned SHARE_LEVELS = (unsigned)(GG_SHARE_LEVELS) & ~3u;
__host__ __device__ constexpr bool level_shared(int s) { return s < 32 && ((SHARE_LEVELS >> s) & 1u); }
// does any of the levels 1 .. steps share?
inline bool any_level_shared(int steps) { return steps >= 2 && (SHARE_LEVELS & ((steps >= 31 ? ~0u : ((2u << steps) - 1u)))) != 0; }

// On a shared level, the walks that stand on one score-cached (hub) node of one root are a group: one warp builds the
// list once and draws every walk of the group from it while the list is still in its score buffer (nothing is stored).
// 0 = hub walks run per walk, as on a level that does not share.  A group of more than HUB_GROUP_MAX walks is split into
// work items that each build the list, so that no single item is the launch's tail.
#ifndef GG_SHARE_HUB
#define GG_SHARE_HUB 1
#endif
#ifndef GG_HUB_GROUP_MAX
#define GG_HUB_GROUP_MAX 128
#endif
constexpr bool SHARE_HUB = GG_SHARE_HUB != 0;
constexpr int HUB_GROUP_MAX = GG_HUB_GROUP_MAX;
static_assert(HUB_GROUP_MAX > 0 && HUB_GROUP_MAX % 32 == 0, "hub work items are whole warps of walks");

template <int CPL>
__global__ void __launch_bounds__(WARPS_PER_CTA * 32, walk_min_ctas(CPL)) walk_kernel(const __grid_constant__ gg_walk_desc d,
                                                                                 const FlatView fv, const int tail_mode) {
    extern __shared__ __align__(16) unsigned char walk_smem[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    float *s_sc = reinterpret_cast<float *>(walk_smem + (size_t)wid * WALK_SMEM_PER_WARP);
    int *s_ids = reinterpret_cast<int *>(s_sc + SC_CAP);
    Stage stg;
    stg.buf = s_sc;
    stg.bar = reinterpret_cast<unsigned long long *>(s_ids + ID_CAP);
    stg.phase = 0u;
    stg.on = !d.no_tma && d.edge_score != nullptr;
    if (stg.on) {
        if (lane == 0) {
            mbar_init(stg.bar, 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncwarp();
    }
    const long long gw = (long long)blockIdx.x * WARPS_PER_CTA + wid;
    int *g_ids = reinterpret_cast<int *>(d.scratch) + (size_t)gw * 2 * (size_t)d.max_cand;
    float *g_sc = reinterpret_cast<float *>(g_ids + d.max_cand);
    Rng rng;
    rng.mode = GG_RNG_PHILOX; rng.k0 = (uint32_t)d.seed; rng.k1 = (uint32_t)(d.seed >> 32); rng.tag = d.pass_tag;
    rng.stream = nullptr; rng.n_stream = 0; rng.cursor = 0; rng.exhausted = 0;
    unsigned long long raw_steps = 0, raw_suml = 0, overflow = 0, rows_gathered = 0;
    unsigned int cyc[7] = {0, 0, 0, 0, 0, 0, 0};
    const bool ratio_all = d.update_ratio >= 1.0;

    const long long n_items = tail_mode ? (long long)fv.ctr[0] : d.n_walks;
    for (;;) {
        unsigned int wi = 0;
        if (lane == 0) wi = atomicAdd(d.work_counter, 1u);
        wi = __shfl_sync(FULL, wi, 0);
        if ((long long)wi >= n_items) break;
        if (tail_mode) {
            // a walk handed over by the level-synchronous steps: continue where it stands
            const int4 rec = fv.tail[wi];
            const long long w = rec.x;
            const int slot = rec.w;
            WalkState from;
            from.cur = rec.y; from.prev = rec.z; from.step = d.wsteps[w]; from.fedge = d.first_edge[w]; from.suml = d.wsuml[w];
            walk_one<CPL>(d, rng, slot, (uint32_t)(w - __ldg(d.walk_ptr + slot)), w, s_ids, s_sc, g_ids, g_sc, lane, raw_steps,
                          raw_suml, overflow, rows_gathered, cyc, stg, &from);
            continue;
        }
        const long long w = d.walk_order ? (long long)__ldg(d.walk_order + wi) : (long long)wi;
        // walk -> root slot: last slot with walk_ptr[slot] <= w (table when the caller provides one)
        int slot;
        if (d.walk_slot) {
            slot = __ldg(d.walk_slot + w);
        } else {
            long long lo = 0, hi = d.n_roots;
            while (hi - lo > 1) {
                const long long mid = (lo + hi) >> 1;
                if (__ldg(d.walk_ptr + mid) <= w) lo = mid; else hi = mid;
            }
            slot = (int)lo;
        }
        const uint32_t k = (uint32_t)(w - __ldg(d.walk_ptr + slot));
        if (!ratio_all) {  // graph_gan.py:189/209: one draw per root
            uint32_t a, b;
            philox4x32_10((uint32_t)d.roots[slot], 0xffffffffu, 0u, rng.tag, rng.k0, rng.k1, a, b);
            if (!(u53(a, b) < d.update_ratio)) {
                if (lane == 0) {
                    d.samples[w] = -1; d.status[w] = GG_SKIPPED; d.first_edge[w] = -1; d.wsteps[w] = 0; d.wsuml[w] = 0;
                    if (d.path_len) d.path_len[w] = 0;
                }
                continue;
            }
        }
        walk_one<CPL>(d, rng, slot, k, w, s_ids, s_sc, g_ids, g_sc, lane, raw_steps, raw_suml, overflow, rows_gathered,
                      cyc, stg);
    }
    if (lane == 0) {
#pragma unroll
        for (int q = 0; q < 7; ++q) if (cyc[q]) atomicAdd(d.counters + GG_CNT_CYC_ENUM + q, (unsigned long long)cyc[q]);
        if (raw_steps) atomicAdd(d.counters + GG_CNT_RAW_STEPS, raw_steps);
        if (raw_suml) atomicAdd(d.counters + GG_CNT_RAW_SUML, raw_suml);
        if (overflow) atomicAdd(d.counters + GG_CNT_PATH_OVERFLOW, overflow);
        if (rows_gathered) atomicAdd(d.counters + GG_CNT_ROWS_GATHERED, rows_gathered);
    }
}

// ---------------------------------------------------------------- level-synchronous ("flat") steps
// The persistent kernel above gives every walk to one warp from root to leaf: per step the warp runs the dependent chain
// indptr -> tree bits / adjacency -> embedding rows -> softmax -> draw alone, so most of the time a resident warp has
// nothing in flight (ncu: 22 cycles per issued instruction, a third of them instruction-cache misses of 32 warps
// scattered over 130 KB of code).  Here all unfinished walks take step s TOGETHER, one phase per kernel:
//   flat_start_kernel   thread per walk: the root step (inverts the root's CDF) and, for (root, child) pairs picked by
//                       several walks, step 1 from the shared CDF (step1_cdf_kernel); survivors enter level 1 or 2
//   flat_enum_kernel    warp per unfinished walk: candidate list [father] + children(cur) from the tree bits into the
//                       item's slab of the id pool (short chain: indptr -> bits + adjacency); empty and single-candidate
//                       lists are finished on the spot; walks standing on a score-cached (hub) node go to the hub list
//   flat_choose_kernel  warp per item: on-demand scores (rows of the candidates: the only phase with row gathers, so
//                       every resident warp has 8 rows in flight almost all the time), softmax + CDF + draw, next
//                       node; hub items run the cached-list step of the persistent kernel (TMA-staged enumeration)
// and after `steps` levels the few walks still alive are finished by walk_kernel in tail mode.  Same arithmetic, same
// Philox counters (root, walk, step): bit-identical to the persistent kernel (tests: test_flat_steps_*).
__device__ __forceinline__ bool step_includes_father(const gg_walk_desc &d, int s, int fedge) {
    if (s == 0) return false;                              // graph_gan.py:250: the root has no father
    if (s == 1) {
        if (d.for_d) return false;                         // graph_gan.py:255-257
        return !((d.d1_bits[fedge >> 5] >> (fedge & 31)) & 1u);   // graph_gan.py:258-259: father entry removed by a D pass
    }
    return true;
}

// the walk made its choice at step s over n candidates: its outputs; true when it goes on (to level s + 1 or the tail)
__device__ __forceinline__ bool flat_record_choice(const gg_walk_desc &d, int s, long long w, int cur, int n, int idx, int nxt,
                                                   bool inc_father, unsigned long long &overflow) {
    if (d.max_path > 0 && d.paths && s + 1 < d.max_path) d.paths[(size_t)w * (size_t)d.max_path + s + 1] = nxt;
    d.wsteps[w] = s + 1;
    d.wsuml[w] = d.wsuml[w] + n;
    if (inc_father && idx == 0) {                          // graph_gan.py:264-266: back to the father: cur is the sample
        d.samples[w] = cur; d.status[w] = GG_DONE;
        if (d.path_len) d.path_len[w] = s + 2;
        if (d.max_path > 0 && s + 2 > d.max_path) overflow += 1;
        return false;
    }
    return true;
}

// lane 0: the walk made its choice at step s over n candidates
__device__ __forceinline__ void flat_advance(const gg_walk_desc &d, const FlatView &fv, int s, long long w, int slot, int cur,
                                             int n, int idx, int nxt, bool inc_father, unsigned long long &overflow) {
    if (flat_record_choice(d, s, w, cur, n, idx, nxt, inc_father, overflow)) {
        const int4 rec = make_int4((int)w, nxt, cur, slot);
        if (s < fv.steps) level_list(fv, s + 1)[atomicAdd(GG_FCTR(fv, s + 1, 0), 1u)] = rec;
        else fv.tail[atomicAdd(fv.ctr, 1u)] = rec;
    }
}
__device__ __forceinline__ void flat_void(const gg_walk_desc &d, int s, long long w) {   // lane 0; graph_gan.py:252-257
    d.samples[w] = -1; d.status[w] = GG_VOID; d.wsteps[w] = s;
    if (d.path_len) d.path_len[w] = 0;
}

__global__ void __launch_bounds__(256) flat_start_kernel(const __grid_constant__ gg_walk_desc d, const FlatView fv) {
    const long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    int dest = 0;                                          // 1 / 2: enters level 1 / 2 (or the tail when there is no such level)
    int4 rec = make_int4(0, 0, 0, 0);
    unsigned steps = 0, suml = 0, over = 0;
    if (w < d.n_walks) {
        const int slot = __ldg(d.walk_slot + w);
        const int root = d.roots[slot];
        const uint32_t k = (uint32_t)(w - __ldg(d.walk_ptr + slot));
        const int fi = d.first_idx[w];                      // root_step_kernel: -2 skipped (update_ratio), -1 isolated root
        int32_t *prow = (d.max_path > 0 && d.paths) ? d.paths + (size_t)w * (size_t)d.max_path : nullptr;
        int sample = -1, status = GG_NOTRUN, fedge = -1, ws = 0, wl = 0, plen = 0;
        if (fi == -2) {
            status = GG_SKIPPED;
        } else {
            if (prow) prow[0] = root;
            if (fi < 0) {
                status = GG_VOID;                           // graph_gan.py:252-253
            } else {
                const long long a0 = d.indptr[root];
                const int n0 = (int)(d.indptr[root + 1] - a0);
                fedge = (int)(a0 + fi);
                const int c = __ldg(d.adj + fedge);
                if (prow && 1 < d.max_path) prow[1] = c;
                ws = 1; wl = n0; steps = 1; suml = (unsigned)n0;
                const long long s1pos = __ldg(d.rq_ptr + slot) + fi;
                if (s1_is_shared(d, s1pos)) {
                    const int n = __ldg(d.s1_n + s1pos);
                    if (n == 0) {
                        status = GG_VOID;                   // graph_gan.py:255-257
                    } else {
                        const bool inc_father = step_includes_father(d, 1, fedge);
                        const long long o = __ldg(d.s1_ptr + s1pos);
                        uint32_t a, b;
                        philox4x32_10((uint32_t)root, k, 1u, d.pass_tag, (uint32_t)d.seed, (uint32_t)(d.seed >> 32), a, b);
                        const int idx = (n == 1) ? 0 : cdf_search_raw(d.s1_q + o, n, u53(a, b));
                        const int nxt = __ldg(d.s1_ids + o + idx);
                        if (prow && 2 < d.max_path) prow[2] = nxt;
                        ws = 2; wl = n0 + n; steps = 2; suml = (unsigned)(n0 + n);
                        if (inc_father && idx == 0) {
                            sample = c; status = GG_DONE; plen = 3;
                            if (d.max_path > 0 && 3 > d.max_path) over = 1;
                        } else {
                            rec = make_int4((int)w, nxt, c, slot); dest = 2;
                        }
                    }
                } else {
                    rec = make_int4((int)w, c, root, slot); dest = 1;
                }
            }
        }
        d.samples[w] = sample; d.status[w] = status; d.first_edge[w] = fedge; d.wsteps[w] = ws; d.wsuml[w] = wl;
        if (d.path_len) d.path_len[w] = plen;
    }
    // warp-aggregated appends (one atomic per warp and destination)
#pragma unroll
    for (int lv = 1; lv <= 2; ++lv) {
        const unsigned mk = __ballot_sync(FULL, dest == lv);
        if (!mk) continue;
        const int leader = __ffs(mk) - 1;
        int4 *list = (lv <= fv.steps) ? fv.list[lv & 1] : fv.tail;
        unsigned *cnt = (lv <= fv.steps) ? GG_FCTR(fv, lv, 0) : fv.ctr;
        unsigned base = 0;
        if (lane == leader) base = atomicAdd(cnt, (unsigned)__popc(mk));
        base = __shfl_sync(FULL, base, leader);
        if (dest == lv) list[base + __popc(mk & ((1u << lane) - 1u))] = rec;
    }
    steps = __reduce_add_sync(FULL, steps); suml = __reduce_add_sync(FULL, suml); over = __reduce_add_sync(FULL, over);
    if (lane == 0) {
        if (steps) atomicAdd(d.counters + GG_CNT_RAW_STEPS, (unsigned long long)steps);
        if (suml) atomicAdd(d.counters + GG_CNT_RAW_SUML, (unsigned long long)suml);
        if (over) atomicAdd(d.counters + GG_CNT_PATH_OVERFLOW, (unsigned long long)over);
    }
}

// ---- shared levels: (1) flat_dedupe_kernel, thread per record: the record's key (root slot, node) goes into the level's
// hash table; the record that inserts a key owns its item (candidate list + CDF).  A key on a score-cached (hub) node is a
// hub group (SHARE_HUB): its owner goes to the hub list, and flat_hub_reserve_kernel + flat_hub_fill_kernel lay out the
// group's records contiguously (without SHARE_HUB, hub records go to the hub list one each and run per walk).
// (2) flat_enum_kernel<true> + flat_choose_kernel<C, true>: the owners' lists and their CDFs; a hub group's warp builds
// its list and draws all its walks at once.  (3) flat_draw_kernel, thread per record: the walk's uniform inverts its
// item's CDF (hub records were drawn in step 2).
__device__ __forceinline__ unsigned long long share_hash(unsigned long long key, unsigned long long mask) {
    return ((key * 0x9E3779B97F4A7C15ull) >> 20) & mask;
}

__global__ void __launch_bounds__(256) flat_dedupe_kernel(const __grid_constant__ gg_walk_desc d, const FlatView fv, const int s) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    const unsigned nA = *GG_FCTR(fv, s, 0);
    if (blockIdx.x * blockDim.x >= nA) return;             // warp-uniform below: whole warps leave together
    bool hub = false, owner = false;
    if (i < nA) {
        const int4 rec = level_list(fv, s)[i];
        const int cur = rec.y, slot = rec.w;
        hub = d.edge_score && (d.indptr[cur + 1] - d.indptr[cur]) >= d.hub_threshold;
        int h = -1;
        if (!hub || SHARE_HUB) {
            const unsigned long long key = (unsigned long long)slot * (unsigned long long)d.n_node + (unsigned long long)cur;
            unsigned long long p = share_hash(key, fv.tbl_mask);
            for (;;) {                                     // linear probing; the table has >= 2 slots per record
                const unsigned long long old = atomicCAS(fv.keys + p, ~0ull, key);
                if (old == ~0ull) { owner = true; fv.owner[p] = (int)i; break; }
                if (old == key) break;
                p = (p + 1) & fv.tbl_mask;
            }
            h = (int)p;
            if (hub) {                                     // a member of the hub group: counted, and negative for flat_draw_kernel
                atomicAdd(fv.gcnt + p, 1u);
                h = -2 - h;
            }
        }
        fv.rec_slot[i] = h;
    }
    const int item = (int)i;
    if (SHARE_HUB) {
        const unsigned mk = __ballot_sync(FULL, hub);
        if (lane == 0 && mk) atomicAdd(GG_FCTR(fv, s, 1), (unsigned)__popc(mk));
        warp_append(hub && owner, fv.hub, GG_FCTR_HUB(fv, s, 0), item, lane);
    } else {
        warp_append(hub, fv.hub, GG_FCTR(fv, s, 1), item, lane);
    }
    warp_append(owner && !hub, fv.uniq, GG_FCTR(fv, s, 2), item, lane);
}

// exclusive offset of this lane's `v` in a range of sum(v) reserved on `cnt` with one atomic per warp
__device__ __forceinline__ unsigned warp_reserve(unsigned v, unsigned *cnt, int lane) {
    unsigned incl = v;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const unsigned x = __shfl_up_sync(FULL, incl, off);
        if (lane >= off) incl += x;
    }
    unsigned base = 0;
    if (lane == 31 && incl) base = atomicAdd(cnt, incl);
    return __shfl_sync(FULL, base, 31) + incl - v;
}

// thread per hub owner: its group's range of hub_rec, and the group's work items (at most HUB_GROUP_MAX walks each)
__global__ void __launch_bounds__(256) flat_hub_reserve_kernel(const FlatView fv, const int s) {
    const unsigned j = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    const unsigned nO = *GG_FCTR_HUB(fv, s, 0);
    if (blockIdx.x * blockDim.x >= nO) return;             // warp-uniform below
    int orec = 0;
    unsigned p = 0, cnt = 0, nw = 0;
    if (j < nO) {
        orec = fv.hub[j];
        p = (unsigned)(-2 - fv.rec_slot[orec]);
        cnt = fv.gcnt[p];
        nw = (cnt + HUB_GROUP_MAX - 1) / HUB_GROUP_MAX;
    }
    const unsigned base = warp_reserve(cnt, GG_FCTR_HUB(fv, s, 2), lane);
    const unsigned it = warp_reserve(nw, GG_FCTR_HUB(fv, s, 1), lane);
    if (j < nO) {
        fv.gpos[p] = base;
        for (unsigned q = 0; q < nw; ++q) {
            const unsigned first = q * HUB_GROUP_MAX;
            fv.hub_work[it + q] = make_int4(orec, (int)(base + first), (int)min(cnt - first, (unsigned)HUB_GROUP_MAX), 0);
        }
    }
}

// thread per record: a hub record takes the next place of its group's range (the order within a group is free: every
// walk draws its own uniform)
__global__ void __launch_bounds__(256) flat_hub_fill_kernel(const FlatView fv, const int s) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= *GG_FCTR(fv, s, 0)) return;
    const int h = fv.rec_slot[i];
    if (h <= -2) fv.hub_rec[atomicAdd(fv.gpos + (-2 - h), 1u)] = (int)i;
}

__global__ void __launch_bounds__(256) flat_draw_kernel(const __grid_constant__ gg_walk_desc d, const FlatView fv, const int s) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    const unsigned nA = *GG_FCTR(fv, s, 0);
    if (blockIdx.x * blockDim.x >= nA) return;
    unsigned long long overflow = 0;
    unsigned steps = 0, suml = 0;
    bool go_on = false;
    int4 rec = make_int4(0, 0, 0, 0);
    if (i < nA) {
        const int h = fv.rec_slot[i];
        if (h >= 0) {                                      // (hub items: done per walk by flat_choose_kernel)
            rec = level_list(fv, s)[i];
            const long long w = rec.x;
            const int cur = rec.y, slot = rec.w;
            const int item = fv.owner[h];
            const int nrec = fv.item_n[item];
            const int n = nrec & 0x3fffffff;
            if (n == 0) {
                flat_void(d, s, w);
            } else {
                const bool inc_father = (nrec >> 30) & 1;
                int idx = 0;
                if (n > 1) {
                    uint32_t a, b;
                    philox4x32_10((uint32_t)d.roots[slot], (uint32_t)(w - __ldg(d.walk_ptr + slot)), (uint32_t)s, d.pass_tag,
                                  (uint32_t)d.seed, (uint32_t)(d.seed >> 32), a, b);
                    idx = cdf_search_raw(fv.pool_cdf + (size_t)item * (size_t)(fv.stride + 1), n, u53(a, b));
                }
                const int nxt = fv.pool_ids[(size_t)item * (size_t)fv.stride + idx];
                go_on = flat_record_choice(d, s, w, cur, n, idx, nxt, inc_father, overflow);
                rec = make_int4((int)w, nxt, cur, slot);
                steps = 1; suml = (unsigned)n;
            }
        }
    }
    if (s < fv.steps) warp_append(go_on, level_list(fv, s + 1), GG_FCTR(fv, s + 1, 0), rec, lane);
    else warp_append(go_on, fv.tail, fv.ctr, rec, lane);
    steps = __reduce_add_sync(FULL, steps); suml = __reduce_add_sync(FULL, suml);
    const unsigned over = __reduce_add_sync(FULL, (unsigned)overflow);
    if (lane == 0) {
        if (steps) atomicAdd(d.counters + GG_CNT_RAW_STEPS, (unsigned long long)steps);
        if (suml) atomicAdd(d.counters + GG_CNT_RAW_SUML, (unsigned long long)suml);
        if (over) atomicAdd(d.counters + GG_CNT_PATH_OVERFLOW, (unsigned long long)over);
    }
}

constexpr int FLAT_ENUM_WARPS = 8;
// SHARED: the level's distinct keys only (fv.uniq, from flat_dedupe_kernel); the item keeps its list length and father flag
// for flat_choose_kernel / flat_draw_kernel and finishes no walk itself
template <bool SHARED>
__global__ void __launch_bounds__(FLAT_ENUM_WARPS * 32, 6) flat_enum_kernel(const __grid_constant__ gg_walk_desc d,
                                                                            const FlatView fv, const int s) {
    const int lane = threadIdx.x & 31;
    const unsigned gw = blockIdx.x * FLAT_ENUM_WARPS + (threadIdx.x >> 5), nwarps = gridDim.x * FLAT_ENUM_WARPS;
    const int4 *A = level_list(fv, s);
    const unsigned nA = SHARED ? *GG_FCTR(fv, s, 2) : *GG_FCTR(fv, s, 0);
    Stage stg;
    stg.buf = nullptr; stg.bar = nullptr; stg.phase = 0u; stg.on = false;
    unsigned long long raw_steps = 0, raw_suml = 0, overflow = 0;
    int4 rec_next = (gw < nA) ? A[SHARED ? fv.uniq[gw] : gw] : make_int4(0, 0, 0, 0);
    for (unsigned j = gw; j < nA; j += nwarps) {
        const unsigned i = SHARED ? (unsigned)fv.uniq[j] : j;
        const int4 rec = rec_next;
        if (j + nwarps < nA) rec_next = A[SHARED ? fv.uniq[j + nwarps] : j + nwarps];   // the next item's record is in flight while this one is enumerated
        const long long w = rec.x;
        const int cur = rec.y, prev = rec.z, slot = rec.w;
        const long long a0 = d.indptr[cur], a1 = d.indptr[cur + 1];
        if (!SHARED && d.edge_score && (a1 - a0) >= d.hub_threshold) {   // score-cached node: the whole step runs in flat_choose_kernel
            if (lane == 0) { fv.hub[atomicAdd(GG_FCTR(fv, s, 1), 1u)] = (int)i; fv.item_n[i] = 0; }
            continue;
        }
        const bool inc_father = step_includes_father(d, s, s == 1 ? d.first_edge[w] : 0);
        const uint32_t *tb = d.tree_bits + (size_t)slot * (size_t)d.tree_words;
        int *ids = fv.pool_ids + (size_t)i * (size_t)fv.stride;
        int n = 0;
        if (inc_father) { if (lane == 0) ids[0] = prev; n = 1; }
        float m = 0.0f;
        enumerate_children<UNR>(d, tb, a0, a1, false, ids, nullptr, lane, n, m, stg);
        __syncwarp();
        if (SHARED) {
            if (lane == 0) fv.item_n[i] = n | (inc_father ? (1 << 30) : 0);
        } else if (n == 0) {
            if (lane == 0) { flat_void(d, s, w); fv.item_n[i] = 0; }
        } else if (n == 1) {
            // softmax = [1.0], cdf = [1.0] and 1.0 > u for every u in [0, 1): index 0, no score, no draw needed
            const int nxt = inc_father ? prev : ids[0];
            if (lane == 0) { flat_advance(d, fv, s, w, slot, cur, 1, 0, nxt, inc_father, overflow); fv.item_n[i] = 0; }
            raw_steps += 1; raw_suml += 1;
        } else if (lane == 0) {
            fv.item_n[i] = n | (inc_father ? (1 << 30) : 0);
        }
    }
    if (lane == 0) {
        if (raw_steps) atomicAdd(d.counters + GG_CNT_RAW_STEPS, raw_steps);
        if (raw_suml) atomicAdd(d.counters + GG_CNT_RAW_SUML, raw_suml);
        if (overflow) atomicAdd(d.counters + GG_CNT_PATH_OVERFLOW, overflow);
    }
}

// SHARED: the items that are not score-cached are the level's distinct keys (fv.uniq); their CDF is stored for
// flat_draw_kernel instead of being drawn from.  Hub items are the same either way.
template <int CPL, bool SHARED>
__global__ void __launch_bounds__(WARPS_PER_CTA * 32, walk_min_ctas(CPL)) flat_choose_kernel(const __grid_constant__ gg_walk_desc d,
                                                                                        const FlatView fv, const int s) {
    extern __shared__ __align__(16) unsigned char walk_smem[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    float *s_sc = reinterpret_cast<float *>(walk_smem + (size_t)wid * WALK_SMEM_PER_WARP);
    int *s_ids = reinterpret_cast<int *>(s_sc + SC_CAP);
    Stage stg;
    stg.buf = s_sc;
    stg.bar = reinterpret_cast<unsigned long long *>(s_ids + ID_CAP);
    stg.phase = 0u;
    stg.on = !d.no_tma && d.edge_score != nullptr;
    if (stg.on) {
        if (lane == 0) {
            mbar_init(stg.bar, 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncwarp();
    }
    const long long gw = (long long)blockIdx.x * WARPS_PER_CTA + wid;
    int *g_ids = reinterpret_cast<int *>(d.scratch) + (size_t)gw * 2 * (size_t)d.max_cand;
    float *g_sc = reinterpret_cast<float *>(g_ids + d.max_cand);
    const int4 *A = level_list(fv, s);
    constexpr bool GROUPS = SHARED && SHARE_HUB;
    const unsigned nA = SHARED ? *GG_FCTR(fv, s, 2) : *GG_FCTR(fv, s, 0);
    const unsigned nH = GROUPS ? *GG_FCTR_HUB(fv, s, 1) : *GG_FCTR(fv, s, 1);
    const uint32_t k0 = (uint32_t)d.seed, k1 = (uint32_t)(d.seed >> 32);
    unsigned long long raw_steps = 0, raw_suml = 0, overflow = 0, rows_gathered = 0;
    unsigned int cyc[7] = {0, 0, 0, 0, 0, 0, 0};
    // work queue: the hub items first, one per pull (they are the long ones); then the other items in chunks of
    // FLAT_CHUNK consecutive list positions per pull, the next item's record and list length in flight while the
    // current one is scored
    constexpr unsigned FLAT_CHUNK = 8;
    const unsigned n_pulls = nH + (nA + FLAT_CHUNK - 1) / FLAT_CHUNK;
    for (;;) {
        unsigned j = 0;
        if (lane == 0) j = atomicAdd(GG_FCTR(fv, s, 3), 1u);
        j = __shfl_sync(FULL, j, 0);
        if (j >= n_pulls) break;
        const bool hub_item = j < nH;
        if (GROUPS && hub_item) {
            // ---- a hub group (or a part of one): the walks of one root on one score-cached node.  From step 2 on their
            // list is [tree father] + children(cur) for all of them; it is built and prepared once, then every walk
            // inverts it with its own uniform: lane t holds the walk of the t-th draw of each round of 32
            const int4 hw = fv.hub_work[j];
            const int4 orec = A[hw.x];
            const int cur = orec.y, prev = orec.z, slot = orec.w;
            const int root = d.roots[slot];
            const long long wp = __ldg(d.walk_ptr + slot);
            int w_lane = (lane < hw.z) ? A[fv.hub_rec[hw.y + lane]].x : 0;      // in flight while the list is built
            const uint32_t *tb = d.tree_bits + (size_t)slot * (size_t)d.tree_words;
            int n; float m; int *ids; float *sc;
            build_list<CPL, UNR>(d, tb, cur, prev, true, s_ids, s_sc, g_ids, g_sc, lane, n, m, ids, sc, rows_gathered, cyc, stg);
            double *tiles = sc != s_sc ? reinterpret_cast<double *>(s_sc) : nullptr;
            ListCdf cdf;
            if (n >= 2) cdf_prepare(sc, n, m, lane, tiles, cdf);
            unsigned long long ov = 0;
            for (int q0 = 0; q0 < hw.z; q0 += 32) {
                if (q0) w_lane = (q0 + lane < hw.z) ? A[fv.hub_rec[hw.y + q0 + lane]].x : 0;
                const int nq = min(32, hw.z - q0);
                const bool mine = lane < nq;
                int idx = 0;                               // n == 1: index 0 for every walk (see build_list)
                if (n >= 2) {
                    // each lane draws the uniform of its own walk; the inversions (warp-wide) run one after the other
                    uint32_t a, b;
                    philox4x32_10((uint32_t)root, (uint32_t)(w_lane - wp), (uint32_t)s, d.pass_tag, k0, k1, a, b);
                    const double u_lane = u53(a, b);
                    for (int t = 0; t < nq; ++t) {
                        const int it = cdf_draw(sc, n, cdf, __shfl_sync(FULL, u_lane, t), lane, tiles);
                        if (lane == t) idx = it;
                    }
                }
                bool go_on = false;
                int4 next = make_int4(0, 0, 0, 0);
                if (mine && n == 0) flat_void(d, s, w_lane);
                if (mine && n > 0) {
                    const int nxt = ids[idx];
                    go_on = flat_record_choice(d, s, w_lane, cur, n, idx, nxt, true, ov);
                    next = make_int4(w_lane, nxt, cur, slot);
                }
                if (s < fv.steps) warp_append(go_on, level_list(fv, s + 1), GG_FCTR(fv, s + 1, 0), next, lane);
                else warp_append(go_on, fv.tail, fv.ctr, next, lane);
                if (lane == 0 && n > 0) { raw_steps += (unsigned)nq; raw_suml += (unsigned)nq * (unsigned)n; }
            }
            const unsigned ovw = __reduce_add_sync(FULL, (unsigned)ov);
            if (lane == 0) overflow += ovw;
            __syncwarp();                                  // every lane is done with ids / sc before the next pull
            continue;
        }
        unsigned p = hub_item ? 0u : (j - nH) * FLAT_CHUNK;
        const unsigned p_end = hub_item ? 1u : ((p + FLAT_CHUNK < nA) ? p + FLAT_CHUNK : nA);
        unsigned i_next = hub_item ? (unsigned)fv.hub[j] : (SHARED ? (unsigned)fv.uniq[p] : p);
        int4 rec_next = A[i_next];
        int n_next = hub_item ? 0 : fv.item_n[i_next];
        for (; p < p_end; ++p) {
            const unsigned i = i_next;
            const int4 rec = rec_next;
            const int nrec = n_next;
            if (p + 1 < p_end) {
                i_next = SHARED ? (unsigned)fv.uniq[p + 1] : p + 1;
                rec_next = A[i_next]; n_next = fv.item_n[i_next];
            }
            if (!hub_item && (nrec & 0x3fffffff) < 2) continue;      // finished by flat_enum_kernel, or a hub item
            const long long w = rec.x;
            const int cur = rec.y, prev = rec.z, slot = rec.w;
            int n, idx, nxt;
            bool inc_father;
            uint32_t a, b;
            if (hub_item) {
                inc_father = step_includes_father(d, s, s == 1 ? d.first_edge[w] : 0);
                const uint32_t *tb = d.tree_bits + (size_t)slot * (size_t)d.tree_words;
                int *ids; float *sc; float m;
                build_list<CPL, UNR>(d, tb, cur, prev, inc_father, s_ids, s_sc, g_ids, g_sc, lane, n, m, ids, sc, rows_gathered, cyc, stg);
                if (n == 0) {
                    if (lane == 0) flat_void(d, s, w);
                    continue;
                }
                philox4x32_10((uint32_t)d.roots[slot], (uint32_t)(w - __ldg(d.walk_ptr + slot)), (uint32_t)s, d.pass_tag, k0, k1, a, b);
                idx = (n == 1) ? 0 : choose_index(sc, n, m, u53(a, b), lane, sc != s_sc ? reinterpret_cast<double *>(s_sc) : nullptr);
                nxt = ids[idx];
                __syncwarp();
            } else {
                n = nrec & 0x3fffffff;
                inc_father = (nrec >> 30) & 1;
                const int *ids = fv.pool_ids + (size_t)i * (size_t)fv.stride;
                float4 c4[CPL];                                          // (ld = 512: the row goes to shared memory)
                float *s_row = CPL == WIDE_CPL ? walk_wide_row(s_sc) : nullptr;
                if constexpr (CPL == WIDE_CPL) load_row_wide(d.emb, d.ld, cur, s_row, lane);
                else load_row<CPL>(d.emb, d.ld, cur, lane & 7, c4);
                const int root = d.roots[slot];
                const uint32_t k = (uint32_t)(w - __ldg(d.walk_ptr + slot));
                if constexpr (CPL == WIDE_CPL) score_list_wide(d.emb, d.bias, d.ld, s_row, ids, s_sc, n, cur, lane);
                else score_list<CPL>(d.emb, d.bias, d.ld, c4, ids, s_sc, n, cur, lane);
                rows_gathered += 1u + (unsigned)n;
                const float m = list_max(s_sc, n, lane);
                if (SHARED) {
                    cdf_store_raw<UNR>(s_sc, n, m, fv.pool_cdf + (size_t)i * (size_t)(fv.stride + 1), lane);
                    __syncwarp();
                    continue;
                }
                philox4x32_10((uint32_t)root, k, (uint32_t)s, d.pass_tag, k0, k1, a, b);
                idx = choose_index(s_sc, n, m, u53(a, b), lane);
                nxt = ids[idx];
                __syncwarp();
            }
            if (lane == 0) {
                flat_advance(d, fv, s, w, slot, cur, n, idx, nxt, inc_father, overflow);
                raw_steps += 1; raw_suml += (unsigned)n;
            }
        }
    }
    if (lane == 0) {
        if (raw_steps) atomicAdd(d.counters + GG_CNT_RAW_STEPS, raw_steps);
        if (raw_suml) atomicAdd(d.counters + GG_CNT_RAW_SUML, raw_suml);
        if (overflow) atomicAdd(d.counters + GG_CNT_PATH_OVERFLOW, overflow);
        if (rows_gathered) atomicAdd(d.counters + GG_CNT_ROWS_GATHERED, rows_gathered);
    }
}

// the layout of desc.flat_buf (host): returns the bytes needed; fills `fv` when `buf` is given
size_t flat_layout(void *buf, long long n_walks, int hub_threshold, int steps, FlatView *fv) {
    const size_t W = (size_t)(n_walks > 0 ? n_walks : 1);
    const int stride = ((hub_threshold > 0 ? hub_threshold : 1) + 31) / 32 * 32;
    size_t off = 0;
    auto take = [&](size_t bytes) {
        void *p = buf ? (void *)((unsigned char *)buf + off) : nullptr;
        off += (bytes + 255) & ~(size_t)255;
        return p;
    };
    unsigned *ctr = (unsigned *)take(sizeof(unsigned) * FLAT_CTR_ALL);
    int4 *l0 = (int4 *)take(16 * W), *l1 = (int4 *)take(16 * W), *tail = (int4 *)take(16 * W);
    int *hub = (int *)take(4 * W), *item_n = (int *)take(4 * W);
    int *pool = (int *)take(4 * W * (size_t)stride);
    // shared levels: a table of >= 2 slots per record (W = 322 k: 2^20 slots, 12 MB), the owners' CDF slab (332 MB); hub
    // groups: a count and a place per table slot (8 MB), the grouped records and the work items (6.4 MB)
    unsigned long long cap = 0;
    unsigned long long *keys = nullptr;
    int *owner = nullptr, *rec_slot = nullptr, *uniq = nullptr, *hub_rec = nullptr;
    unsigned *gcnt = nullptr, *gpos = nullptr;
    int4 *hub_work = nullptr;
    double *cdf = nullptr;
    if (any_level_shared(steps)) {
        cap = 1;
        while (cap < 2 * (unsigned long long)W) cap <<= 1;
        keys = (unsigned long long *)take(8 * cap);
        owner = (int *)take(4 * cap);
        rec_slot = (int *)take(4 * W);
        uniq = (int *)take(4 * W);
        cdf = (double *)take(8 * W * (size_t)(stride + 1));
        if (SHARE_HUB) {
            gcnt = (unsigned *)take(4 * cap);
            gpos = (unsigned *)take(4 * cap);
            hub_rec = (int *)take(4 * W);
            hub_work = (int4 *)take(16 * W);
        }
    }
    if (fv) {
        fv->ctr = ctr; fv->list[0] = l0; fv->list[1] = l1; fv->tail = tail; fv->hub = hub;
        fv->item_n = item_n; fv->pool_ids = pool; fv->stride = stride; fv->steps = steps;
        fv->keys = keys; fv->owner = owner; fv->rec_slot = rec_slot; fv->uniq = uniq; fv->pool_cdf = cdf;
        fv->tbl_mask = cap ? cap - 1 : 0;
        fv->gcnt = gcnt; fv->gpos = gpos; fv->hub_rec = hub_rec; fv->hub_work = hub_work;
    }
    return off;
}

// ---------------------------------------------------------------- reference-order (stream) kernel
// One warp replays the reference's sequential consumption of a uniform stream: a draw per
// root (graph_gan.py:189/209), a draw per choice (:262), stop at a root's first void.  (ld = 512: one CTA per SM is
// declared so that ptxas gives the kernel the registers of the streamed candidate row instead of spilling it.)
template <int CPL>
__global__ void __launch_bounds__(32, CPL == WIDE_CPL ? 1 : 0) walk_stream_kernel(const __grid_constant__ gg_walk_desc d) {
    extern __shared__ __align__(16) unsigned char walk_smem[];
    float *s_sc = reinterpret_cast<float *>(walk_smem);
    int *s_ids = reinterpret_cast<int *>(s_sc + SC_CAP);
    const int lane = threadIdx.x;
    int *g_ids = reinterpret_cast<int *>(d.scratch);
    float *g_sc = reinterpret_cast<float *>(g_ids + d.max_cand);
    Rng rng;
    rng.mode = GG_RNG_STREAM; rng.k0 = rng.k1 = rng.tag = 0;
    rng.stream = d.stream; rng.n_stream = d.n_stream; rng.cursor = 0; rng.exhausted = 0;
    unsigned long long raw_steps = 0, raw_suml = 0, overflow = 0, rows_gathered = 0;
    unsigned int cyc[7] = {0, 0, 0, 0, 0, 0, 0};
    Stage stg;                                              // the replay kernel uses plain loads
    stg.buf = s_sc; stg.bar = nullptr; stg.phase = 0u; stg.on = false;
    for (long long slot = 0; slot < d.n_roots && !rng.exhausted; ++slot) {
        const long long w0 = d.walk_ptr[slot], w1 = d.walk_ptr[slot + 1];
        const double ur = rng.draw(0, 0, 0);
        const bool skip = !(ur < d.update_ratio);
        bool dead = skip || rng.exhausted;
        for (long long w = w0; w < w1; ++w) {
            if (dead) {
                if (lane == 0) {
                    d.samples[w] = -1; d.status[w] = skip ? GG_SKIPPED : GG_NOTRUN; d.first_edge[w] = -1;
                    d.wsteps[w] = 0; d.wsuml[w] = 0;
                    if (d.path_len) d.path_len[w] = 0;
                }
                continue;
            }
            const int st = walk_one<CPL>(d, rng, (int)slot, (uint32_t)(w - w0), w, s_ids, s_sc, g_ids, g_sc, lane,
                                         raw_steps, raw_suml, overflow, rows_gathered, cyc, stg);
            if (st != GG_DONE) dead = true;
        }
    }
    if (lane == 0) {
        atomicAdd(d.counters + GG_CNT_RAW_STEPS, raw_steps);
        atomicAdd(d.counters + GG_CNT_RAW_SUML, raw_suml);
        atomicAdd(d.counters + GG_CNT_PATH_OVERFLOW, overflow);
        atomicAdd(d.counters + GG_CNT_ROWS_GATHERED, rows_gathered);
        d.counters[GG_CNT_STREAM_USED] = (unsigned long long)rng.cursor + (rng.exhausted ? (1ull << 62) : 0ull);
    }
}

// ---------------------------------------------------------------- finalize (thread per walk)
// Three flat passes instead of one warp per root (a hub root has > 10 k walks: its warp was the launch's tail):
//   1. every walk that is not DONE lowers its root's "first bad walk" (atomicMin into root_ok, used as scratch)
//   2. every walk up to and including the first bad one adds its counters and (D mode) its father-removal bit;
//      the walks after it are blanked -- the reference never ran them (graph_gan.py:252-257 returned early)
//   3. per root: root_ok = no bad walk and at least one walk ("neg is not None and len(pos) != 0", graph_gan.py:192)
constexpr int FIN_NONE = 0x7f7f7f7f;                      // (the memset pattern root_ok is initialised with)

__device__ __forceinline__ long long walk_root_slot(const long long *__restrict__ walk_ptr, long long n_roots, long long w) {
    long long lo = 0, hi = n_roots;                         // last slot with walk_ptr[slot] <= w
    while (hi - lo > 1) {
        const long long mid = (lo + hi) >> 1;
        if (__ldg(walk_ptr + mid) <= w) lo = mid; else hi = mid;
    }
    return lo;
}

__global__ void finalize_mark_kernel(long long n_roots, const long long *__restrict__ walk_ptr, const int *__restrict__ status,
                                     int *root_ok) {
    const long long W = walk_ptr[n_roots];
    for (long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x; w < W; w += (long long)gridDim.x * blockDim.x) {
        if (status[w] == GG_DONE) continue;
        const long long slot = walk_root_slot(walk_ptr, n_roots, w);
        atomicMin(root_ok + slot, (int)(w - walk_ptr[slot]));
    }
}

__global__ void finalize_apply_kernel(long long n_roots, const long long *__restrict__ walk_ptr, int for_d, int *samples,
                                      int *status, const int *__restrict__ first_edge, int *wsteps, int *wsuml, int *path_len,
                                      uint32_t *d1_bits, const int *__restrict__ root_ok, unsigned long long *counters) {
    const long long W = walk_ptr[n_roots];
    unsigned long long steps = 0, suml = 0;
    for (long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x; w < W; w += (long long)gridDim.x * blockDim.x) {
        const long long slot = walk_root_slot(walk_ptr, n_roots, w);
        const long long off = w - walk_ptr[slot];
        if (off <= (long long)root_ok[slot]) {
            steps += (unsigned)wsteps[w]; suml += (unsigned)wsuml[w];
            if (for_d && status[w] == GG_DONE) {
                const int fe = first_edge[w];
                if (fe >= 0) atomicOr(d1_bits + (fe >> 5), 1u << (fe & 31));
            }
        } else {
            if (status[w] != GG_SKIPPED) status[w] = GG_NOTRUN;
            samples[w] = -1; wsteps[w] = 0; wsuml[w] = 0;
            if (path_len) path_len[w] = 0;
        }
    }
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
        steps += __shfl_xor_sync(FULL, steps, off);
        suml += __shfl_xor_sync(FULL, suml, off);
    }
    if ((threadIdx.x & 31) == 0) {
        if (steps) atomicAdd(counters + GG_CNT_STEPS, steps);
        if (suml) atomicAdd(counters + GG_CNT_SUML, suml);
    }
}

__global__ void finalize_roots_kernel(long long n_roots, const long long *__restrict__ walk_ptr, int *root_ok,
                                      unsigned long long *counters) {
    const long long slot = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long acc = 0, okr = 0;
    if (slot < n_roots) {
        const long long k = walk_ptr[slot + 1] - walk_ptr[slot];
        const bool ok = root_ok[slot] == FIN_NONE && k > 0;
        root_ok[slot] = ok ? 1 : 0;
        if (ok) { acc = (unsigned long long)k; okr = 1; }
    }
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
        acc += __shfl_xor_sync(FULL, acc, off);
        okr += __shfl_xor_sync(FULL, okr, off);
    }
    if ((threadIdx.x & 31) == 0 && okr) {
        atomicAdd(counters + GG_CNT_ACCEPTED, acc);
        atomicAdd(counters + GG_CNT_OK_ROOTS, okr);
    }
}

// ---------------------------------------------------------------- D rows
__global__ void row_count_kernel(long long n_roots, const long long *walk_ptr, const int *root_ok, long long *row_ptr) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_roots) row_ptr[i] = root_ok[i] ? 2 * (walk_ptr[i + 1] - walk_ptr[i]) : 0;
}

// thread per walk: its positive row and its negative row (graph_gan.py:194-201)
__global__ void emit_rows_kernel(long long n_roots, const int *__restrict__ roots, const long long *__restrict__ walk_ptr,
                                 const long long *__restrict__ pos_indptr, const int *__restrict__ pos_flat,
                                 const int *__restrict__ root_ok, const int *__restrict__ samples,
                                 const long long *__restrict__ row_ptr, int *center, int *neighbor, int *label) {
    const long long W = walk_ptr[n_roots];
    for (long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x; w < W; w += (long long)gridDim.x * blockDim.x) {
        const long long slot = walk_root_slot(walk_ptr, n_roots, w);
        if (!root_ok[slot]) continue;
        const int r = roots[slot];
        const long long w0 = walk_ptr[slot], k = walk_ptr[slot + 1] - w0, t = w - w0, o = row_ptr[slot];
        center[o + t] = r; neighbor[o + t] = pos_flat[pos_indptr[r] + t]; label[o + t] = 1;
        center[o + k + t] = r; neighbor[o + k + t] = samples[w]; label[o + k + t] = 0;
    }
}

int grid_ctas() { return sm_count() * WALK_MIN_CTAS; }
// CTAs of a walk kernel launch (ld = 512: fewer per SM, so never more than grid_ctas(), which sizes the scratch)
int walk_ctas(int cpl) { return sm_count() * walk_min_ctas(cpl); }
static_assert(WIDE_MIN_CTAS <= WALK_MIN_CTAS, "the walk scratch is sized for grid_ctas() warps");

}  // namespace
}  // namespace gg

extern "C" int gg_walk_scratch_bytes(int32_t max_cand, int64_t *bytes) {
    GG_REQUIRE(bytes && max_cand > 0, "bad arguments");
    const int64_t warps = (int64_t)gg::grid_ctas() * gg::WARPS_PER_CTA;
    *bytes = warps * 2 * (int64_t)max_cand * 4;
    return 0;
}

extern "C" int gg_walk_flat_bytes(int64_t n_walks, int32_t hub_threshold, int32_t flat_steps, int64_t *bytes) {
    GG_REQUIRE(bytes && n_walks >= 0 && hub_threshold > 0 && flat_steps >= 0 && flat_steps <= gg::FLAT_MAX_STEPS, "bad arguments");
    *bytes = (int64_t)gg::flat_layout(nullptr, n_walks, hub_threshold, flat_steps, nullptr);
    return 0;
}

extern "C" int gg_walk_sample(const gg_walk_desc *dp, void *stream) {
    GG_REQUIRE(dp, "null descriptor");
    const gg_walk_desc &d = *dp;
    GG_REQUIRE(gg::ld_supported(d.ld), GG_LD_MESSAGE);
    if (d.n_walks == 0 || d.n_roots == 0) return 0;   // nothing to do (empty batches carry null pointers)
    GG_REQUIRE(d.emb && d.bias && d.indptr && d.adj && d.roots && d.tree_bits && d.walk_ptr, "null graph/embedding pointer");
    GG_REQUIRE(d.tree_words > 0, "tree_words missing (gg_tree_words)");
    GG_REQUIRE(d.samples && d.status && d.first_edge && d.wsteps && d.wsuml && d.counters && d.work_counter,
               "null output pointer");
    GG_REQUIRE(d.for_d || d.d1_bits, "G mode needs d1_bits");
    GG_REQUIRE(d.n_walks < (1ll << 32), "too many walks in one call");
    GG_REQUIRE(d.max_cand > 0 && d.scratch, "scratch missing");
    GG_REQUIRE(!d.root_q || d.rq_ptr, "root_q needs rq_ptr");
    // optional groups: all of a group or none of it (a half-filled descriptor is an argument error, not a fault)
    GG_REQUIRE(d.max_path >= 0 && (d.max_path == 0 || (d.paths && d.path_len)), "max_path > 0 needs paths and path_len");
    GG_REQUIRE(d.phase_mask >= 0 && d.phase_mask <= 3, "phase_mask must be 0..3");
    GG_REQUIRE(d.update_ratio >= 0.0, "update_ratio must be >= 0");
    GG_REQUIRE(d.rng_mode == GG_RNG_PHILOX || d.rng_mode == GG_RNG_STREAM, "unknown rng_mode");
    {
        const bool any_s1 = d.s1_q || d.s1_ids || d.s1_cnt || d.s1_n || d.s1_ptr || d.s1_slot || d.first_idx || d.s1_order;
        GG_REQUIRE(!any_s1 || (d.s1_q && d.s1_ids && d.s1_cnt && d.s1_n && d.s1_ptr && d.s1_slot && d.first_idx && d.s1_nq > 0),
                   "depth-1 reuse: s1_q, s1_ids, s1_cnt, s1_n, s1_ptr, s1_slot, first_idx and s1_nq go together");
        GG_REQUIRE(!any_s1 || d.rng_mode == GG_RNG_PHILOX, "depth-1 reuse needs GG_RNG_PHILOX");
        GG_REQUIRE(!d.walk_order || d.rng_mode == GG_RNG_PHILOX, "walk_order needs GG_RNG_PHILOX");
    }
    GG_REQUIRE(!d.edge_score || (d.hub_threshold > 0 && d.hub_threshold < gg::SMEM_CAP), "hub_threshold out of range");
    cudaStream_t st = (cudaStream_t)stream;
    GG_CHECK(cudaMemsetAsync(d.work_counter, 0, sizeof(unsigned int), st));
    if (d.n_walks == 0 || d.n_roots == 0) return 0;
    const int cpl = d.ld / 32;
    if (d.rng_mode == GG_RNG_STREAM) {
        GG_REQUIRE(d.stream, "stream mode needs the uniform stream");
        GG_REQUIRE(d.scratch_bytes >= 2ll * d.max_cand * 4, "scratch too small");
        switch (cpl) {
#define GG_STREAM(C)                                                                                                  \
    GG_CHECK(cudaFuncSetAttribute(gg::walk_stream_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize,            \
                                  gg::walk_smem_bytes(C, 1)));                                                       \
    gg::walk_stream_kernel<C><<<1, 32, gg::walk_smem_bytes(C, 1), st>>>(d)
            case 1: GG_STREAM(1); break;
            case 2: GG_STREAM(2); break;
            case 4: GG_STREAM(4); break;
            case 8: GG_STREAM(8); break;
            case 16: GG_STREAM(16); break;
#undef GG_STREAM
            default: gg::set_error("gg_walk_sample: unsupported ld %d (supported: 32, 64, 128, 256, 512)", d.ld); return 2;
        }
    } else {
        const int ctas = gg::grid_ctas();
        GG_REQUIRE(d.scratch_bytes >= (int64_t)ctas * gg::WARPS_PER_CTA * 2 * d.max_cand * 4, "scratch too small");
        const int pm = d.phase_mask ? d.phase_mask : 3;   // 1 = depth-1 precompute, 2 = walk kernel (default both)
        if (d.s1_q && (pm & 1)) {   // depth-1 reuse: root steps + one CDF per (root, child) pair that occurs
            GG_REQUIRE(d.root_q && d.walk_slot && d.first_idx && d.s1_cnt && d.s1_n && d.s1_ptr && d.s1_ids && d.s1_slot,
                       "depth-1 reuse needs root_q, walk_slot and the s1_* buffers");
            GG_CHECK(cudaMemsetAsync(d.s1_cnt, 0, sizeof(int32_t) * (size_t)d.s1_nq, st));
            gg::root_step_kernel<<<(unsigned)((d.n_walks + 255) / 256), 256, 0, st>>>(d);
            GG_CHECK(cudaGetLastError());
#define GG_S1(C)                                                                                                      \
    GG_CHECK(cudaFuncSetAttribute(gg::step1_cdf_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize,              \
                                  gg::walk_smem_bytes(C, gg::WARPS_PER_CTA)));                                      \
    gg::step1_cdf_kernel<C><<<gg::walk_ctas(C), gg::WARPS_PER_CTA * 32, gg::walk_smem_bytes(C, gg::WARPS_PER_CTA), st>>>(d)
            switch (cpl) {
                case 1: GG_S1(1); break;
                case 2: GG_S1(2); break;
                case 4: GG_S1(4); break;
                case 8: GG_S1(8); break;
            case 16: GG_S1(16); break;
                default: gg::set_error("gg_walk_sample: unsupported ld %d (supported: 32, 64, 128, 256, 512)", d.ld); return 2;
            }
#undef GG_S1
            GG_CHECK(cudaGetLastError());
            GG_CHECK(cudaMemsetAsync(d.work_counter, 0, sizeof(unsigned int), st));   // the walk kernel's queue starts at 0
        }
        if (!(pm & 2)) return 0;
        gg::FlatView fv;
        memset(&fv, 0, sizeof(fv));
        int tail_mode = 0;
        if (d.flat_steps > 0) {
            // level-synchronous steps (flat_*_kernel), then the persistent kernel finishes what is left
            GG_REQUIRE(d.s1_q && d.edge_score && d.root_q && d.walk_slot && d.first_idx, "flat_steps needs the depth-1 reuse (s1_*, edge_score, root_q, walk_slot)");
            GG_REQUIRE(d.flat_steps <= gg::FLAT_MAX_STEPS, "flat_steps too large");
            GG_REQUIRE(d.flat_buf && d.flat_bytes >= (int64_t)gg::flat_layout(nullptr, d.n_walks, d.hub_threshold, d.flat_steps, nullptr),
                       "flat_buf too small (gg_walk_flat_bytes)");
            gg::flat_layout(d.flat_buf, d.n_walks, d.hub_threshold, d.flat_steps, &fv);
            GG_CHECK(cudaMemsetAsync(fv.ctr, 0, sizeof(unsigned) * gg::FLAT_CTR_ALL, st));
            gg::flat_start_kernel<<<(unsigned)((d.n_walks + 255) / 256), 256, 0, st>>>(d, fv);
            GG_CHECK(cudaGetLastError());
            const int enum_ctas = gg::sm_count() * 8;
            const unsigned rec_ctas = (unsigned)((d.n_walks + 255) / 256);
            GG_REQUIRE(!gg::any_level_shared(d.flat_steps) || d.n_node > 0, "n_node missing");
            for (int s = 1; s <= d.flat_steps; ++s) {
                const bool shared = gg::level_shared(s);
                if (shared) {
                    GG_CHECK(cudaMemsetAsync(fv.keys, 0xff, sizeof(unsigned long long) * (size_t)(fv.tbl_mask + 1), st));
                    if (gg::SHARE_HUB) GG_CHECK(cudaMemsetAsync(fv.gcnt, 0, sizeof(unsigned) * (size_t)(fv.tbl_mask + 1), st));
                    gg::flat_dedupe_kernel<<<rec_ctas, 256, 0, st>>>(d, fv, s);
                    GG_CHECK(cudaGetLastError());
                    if (gg::SHARE_HUB) {
                        gg::flat_hub_reserve_kernel<<<rec_ctas, 256, 0, st>>>(fv, s);
                        GG_CHECK(cudaGetLastError());
                        gg::flat_hub_fill_kernel<<<rec_ctas, 256, 0, st>>>(fv, s);
                        GG_CHECK(cudaGetLastError());
                    }
                    gg::flat_enum_kernel<true><<<enum_ctas, gg::FLAT_ENUM_WARPS * 32, 0, st>>>(d, fv, s);
                } else {
                    gg::flat_enum_kernel<false><<<enum_ctas, gg::FLAT_ENUM_WARPS * 32, 0, st>>>(d, fv, s);
                }
                GG_CHECK(cudaGetLastError());
                switch (cpl) {
#define GG_FLAT(C)                                                                                                    \
    if (shared) {                                                                                                    \
        GG_CHECK(cudaFuncSetAttribute(gg::flat_choose_kernel<C, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,  \
                                      gg::walk_smem_bytes(C, gg::WARPS_PER_CTA)));                                  \
        gg::flat_choose_kernel<C, true><<<gg::walk_ctas(C), gg::WARPS_PER_CTA * 32, gg::walk_smem_bytes(C, gg::WARPS_PER_CTA), st>>>(d, fv, s); \
    } else {                                                                                                         \
        GG_CHECK(cudaFuncSetAttribute(gg::flat_choose_kernel<C, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                      gg::walk_smem_bytes(C, gg::WARPS_PER_CTA)));                                  \
        gg::flat_choose_kernel<C, false><<<gg::walk_ctas(C), gg::WARPS_PER_CTA * 32, gg::walk_smem_bytes(C, gg::WARPS_PER_CTA), st>>>(d, fv, s); \
    }
                    case 1: GG_FLAT(1); break;
                    case 2: GG_FLAT(2); break;
                    case 4: GG_FLAT(4); break;
                    case 8: GG_FLAT(8); break;
            case 16: GG_FLAT(16); break;
#undef GG_FLAT
                    default: gg::set_error("gg_walk_sample: unsupported ld %d (supported: 32, 64, 128, 256, 512)", d.ld); return 2;
                }
                GG_CHECK(cudaGetLastError());
                if (shared) {
                    gg::flat_draw_kernel<<<rec_ctas, 256, 0, st>>>(d, fv, s);
                    GG_CHECK(cudaGetLastError());
                }
            }
            tail_mode = 1;
        }
        switch (cpl) {
#define GG_WALK(C)                                                                                                    \
    GG_CHECK(cudaFuncSetAttribute(gg::walk_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize,                   \
                                  gg::walk_smem_bytes(C, gg::WARPS_PER_CTA)));                                      \
    gg::walk_kernel<C><<<gg::walk_ctas(C), gg::WARPS_PER_CTA * 32, gg::walk_smem_bytes(C, gg::WARPS_PER_CTA), st>>>(d, fv, tail_mode)
            case 1: GG_WALK(1); break;
            case 2: GG_WALK(2); break;
            case 4: GG_WALK(4); break;
            case 8: GG_WALK(8); break;
            case 16: GG_WALK(16); break;
#undef GG_WALK
            default: gg::set_error("gg_walk_sample: unsupported ld %d (supported: 32, 64, 128, 256, 512)", d.ld); return 2;
        }
    }
    return gg::check_cuda(cudaGetLastError(), "walk kernel launch");
}

extern "C" int gg_walk_finalize(int64_t n_roots, const int64_t *walk_ptr, int32_t for_d, int32_t *samples,
                                int32_t *status, const int32_t *first_edge, int32_t *wsteps, int32_t *wsuml,
                                int32_t *path_len, uint32_t *d1_bits, int32_t *root_ok,
                                unsigned long long *counters, void *stream) {
    GG_REQUIRE(walk_ptr && samples && status && first_edge && wsteps && wsuml && root_ok && counters, "null pointer");
    GG_REQUIRE(!for_d || d1_bits, "D mode needs d1_bits");
    if (n_roots == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    const int threads = 256;
    const unsigned wgrid = (unsigned)(gg::sm_count() * 8);           // grid-stride over the walks (their number is on the device)
    GG_CHECK(cudaMemsetAsync(root_ok, 0x7f, sizeof(int32_t) * (size_t)n_roots, st));
    gg::finalize_mark_kernel<<<wgrid, threads, 0, st>>>(n_roots, (const long long *)walk_ptr, status, root_ok);
    GG_CHECK(cudaGetLastError());
    gg::finalize_apply_kernel<<<wgrid, threads, 0, st>>>(n_roots, (const long long *)walk_ptr, for_d, samples, status, first_edge,
                                                        wsteps, wsuml, path_len, d1_bits, root_ok, counters);
    GG_CHECK(cudaGetLastError());
    gg::finalize_roots_kernel<<<(unsigned)((n_roots + threads - 1) / threads), threads, 0, st>>>(
        n_roots, (const long long *)walk_ptr, root_ok, counters);
    return gg::check_cuda(cudaGetLastError(), "finalize kernel launch");
}

extern "C" int gg_emit_d_rows(int64_t n_roots, const int32_t *roots, const int64_t *walk_ptr,
                              const int64_t *pos_indptr, const int32_t *pos_flat, const int32_t *root_ok,
                              const int32_t *samples, int64_t *row_ptr, int32_t *center, int32_t *neighbor,
                              int32_t *label, int64_t *n_rows_out, void *stream) {
    GG_REQUIRE(row_ptr && n_rows_out, "null pointer");
    GG_REQUIRE(n_roots == 0 || (roots && walk_ptr && pos_indptr && pos_flat && root_ok && samples), "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const int threads = 256;
    if (n_roots > 0) {
        gg::row_count_kernel<<<(unsigned)((n_roots + threads - 1) / threads), threads, 0, st>>>(
            n_roots, (const long long *)walk_ptr, root_ok, (long long *)row_ptr);
        GG_CHECK(cudaGetLastError());
    }
    int rc = gg::launch_exclusive_scan_i64((long long *)row_ptr, n_roots, (long long *)n_rows_out, st);
    if (rc) return rc;
    if (n_roots == 0) return 0;
    GG_REQUIRE(center && neighbor && label, "null output pointer");
    gg::emit_rows_kernel<<<(unsigned)(gg::sm_count() * 8), threads, 0, st>>>(n_roots, roots, (const long long *)walk_ptr,
                                                               (const long long *)pos_indptr, pos_flat, root_ok,
                                                               samples, (const long long *)row_ptr, center, neighbor,
                                                               label);
    return gg::check_cuda(cudaGetLastError(), "emit rows launch");
}
