// walk_list.cuh -- the candidate list of a walk step (graph_gan.py:250-259), shared by the walk sampler (walk.cu) and
// the exact generator distribution (gdist.cu): children enumerated from the tree bits, on-demand or cached scores.
#pragma once
#include "walk_common.cuh"

namespace gg {

// children of `cur` among its walk-CSR entries [a0, a1): the set bits of the root's tree row `tb` (csrc/bfs.cu), in
// entry order == adjacency order == the reference's list order (graph_gan.py:102-105).  One coalesced load brings 32
// bitmap words (1024 entries); only words with a set bit touch adj[] / edge_score[], U of them in flight.
template <int U>
__device__ __forceinline__ void enumerate_children(const gg_walk_desc &d, const uint32_t *__restrict__ tb, long long a0,
                                                   long long a1, bool cached, int *ids, float *sc, int lane, int &n, float &m,
                                                   Stage &stg) {
    if (a1 <= a0) return;
    const unsigned lt = (1u << lane) - 1u;
    if (a1 - a0 <= 64) {
        // short list (the common case): adjacency entries and their bitmap words are loaded together -- the step's
        // dependent chain is indptr -> {bits, adj} -> rows instead of indptr -> bits -> adj -> rows
        const long long e0 = a0 + lane, e1 = a0 + 32 + lane;
        const bool in0 = e0 < a1, in1 = e1 < a1;
        const unsigned w0 = in0 ? __ldg(tb + (e0 >> 5)) : 0u, w1 = in1 ? __ldg(tb + (e1 >> 5)) : 0u;
        const int v0 = in0 ? __ldg(d.adj + e0) : -1, v1 = in1 ? __ldg(d.adj + e1) : -1;
        const float c0 = (cached && in0) ? __ldg(d.edge_score + e0) : 0.0f, c1 = (cached && in1) ? __ldg(d.edge_score + e1) : 0.0f;
        const bool s0 = in0 && ((w0 >> (e0 & 31)) & 1u), s1 = in1 && ((w1 >> (e1 & 31)) & 1u);
        const unsigned m0 = __ballot_sync(FULL, s0), m1 = __ballot_sync(FULL, s1);
        if (s0) {
            const int pos = n + __popc(m0 & lt);
            ids[pos] = v0;
            if (cached) { sc[pos] = c0; m = fmaxf(m, c0); }
        }
        n += __popc(m0);
        if (s1) {
            const int pos = n + __popc(m1 & lt);
            ids[pos] = v1;
            if (cached) { sc[pos] = c1; m = fmaxf(m, c1); }
        }
        n += __popc(m1);
        return;
    }
    const long long wfirst = a0 >> 5, wlast = (a1 - 1) >> 5;
    if (cached && stg.on && (a1 - a0 + 1) > SC_CAP) {
        // ---- hub list, TMA staged: the list is longer than the warp's shared score buffer, so its scores go to the
        // global scratch and the buffer is idle: each 512-entry block of adj[] and edge_score[] (contiguous, 128-B
        // aligned) is brought in by ONE elected lane with two cp.async.bulk copies completing on the warp's mbarrier --
        // one round trip per 512 entries instead of one per 128 -- while the lanes fetch the block's 16 bitmap words.
        int *s_adj = reinterpret_cast<int *>(stg.buf);
        float *s_cs = stg.buf + STAGE_ENTRIES;
        const long long a1r = (a1 + 3) & ~3ll;                      // copy sizes are multiples of 16 bytes (arrays are padded)
        for (long long eb = wfirst << 5; eb < a1; eb += STAGE_ENTRIES) {
            const unsigned bytes = (unsigned)(((eb + STAGE_ENTRIES < a1r) ? (long long)STAGE_ENTRIES : (a1r - eb)) * 4);
            if (lane == 0) {
                mbar_expect_tx(stg.bar, 2 * bytes);
                bulk_g2s(s_adj, d.adj + eb, bytes, stg.bar);
                bulk_g2s(s_cs, d.edge_score + eb, bytes, stg.bar);
            }
            const long long wi = (eb >> 5) + lane;
            unsigned word = (lane < STAGE_ENTRIES / 32 && wi <= wlast) ? __ldg(tb + wi) : 0u;
            if (wi == wfirst) word &= 0xffffffffu << (a0 & 31);
            if (wi == wlast && (a1 & 31)) word &= (1u << (a1 & 31)) - 1u;
            unsigned nz = __ballot_sync(FULL, word != 0u);
            mbar_wait(stg.bar, stg.phase);
            stg.phase ^= 1u;
            while (nz) {
                const int j = __ffs(nz) - 1;
                nz &= nz - 1u;
                const unsigned wv = __shfl_sync(FULL, word, j);
                if ((wv >> lane) & 1u) {
                    const int pos = n + __popc(wv & lt);
                    const float cs = s_cs[32 * j + lane];
                    ids[pos] = s_adj[32 * j + lane];
                    sc[pos] = cs;
                    m = fmaxf(m, cs);
                }
                n += __popc(wv);
            }
            __syncwarp();                                           // every lane is done with the block before it is overwritten
        }
        return;
    }
    for (long long wb = wfirst; wb <= wlast; wb += 32) {
        const long long wi = wb + lane;
        unsigned word = (wi <= wlast) ? __ldg(tb + wi) : 0u;
        if (wi == wfirst) word &= 0xffffffffu << (a0 & 31);
        if (wi == wlast && (a1 & 31)) word &= (1u << (a1 & 31)) - 1u;
        unsigned nz = __ballot_sync(FULL, word != 0u);
        while (nz) {
            int jw[U], v[U];
            unsigned wv[U];
            float cs[U];
#pragma unroll
            for (int k = 0; k < U; ++k) {
                jw[k] = nz ? (__ffs(nz) - 1) : -1;
                nz &= nz - 1u;                              // 0 & 0xffffffff == 0: stays empty
            }
#pragma unroll
            for (int k = 0; k < U; ++k) {
                const unsigned x = __shfl_sync(FULL, word, jw[k] & 31);
                wv[k] = (jw[k] >= 0) ? x : 0u;
            }
#pragma unroll
            for (int k = 0; k < U; ++k) {
                const bool isc = (wv[k] >> lane) & 1u;
                const long long e = ((wb + jw[k]) << 5) + lane;
                v[k] = isc ? __ldg(d.adj + e) : -1;
                cs[k] = (cached && isc) ? __ldg(d.edge_score + e) : 0.0f;
            }
#pragma unroll
            for (int k = 0; k < U; ++k) {
                if (jw[k] < 0) break;                       // warp-uniform
                if ((wv[k] >> lane) & 1u) {
                    const int pos = n + __popc(wv[k] & lt);
                    ids[pos] = v[k];
                    if (cached) { sc[pos] = cs[k]; m = fmaxf(m, cs[k]); }
                }
                n += __popc(wv[k]);
            }
        }
    }
}

// Candidate list of `cur` in the tree of the root whose tree row is `tb` (graph_gan.py:250-259):
// [father] + children in adjacency order, with scores all_score[cur, cand] (generator.py:21) -- cached hub
// scores or the on-demand canonical dot -- and their max.  Warp-cooperative; results are warp-uniform.
template <int CPL, int U>
__device__ __forceinline__ void build_list(const gg_walk_desc &d, const uint32_t *__restrict__ tb, int cur, int prev,
                                           bool inc_father, int *s_ids, float *s_sc, int *g_ids, float *g_sc, int lane,
                                           int &n_out, float &m_out, int *&ids_out, float *&sc_out,
                                           unsigned long long &rows_gathered, unsigned int (&cyc)[7], Stage &stg) {
    const long long a0 = d.indptr[cur], a1 = d.indptr[cur + 1];
    const bool cached = d.edge_score && (a1 - a0) >= d.hub_threshold;  // scores precomputed per pass
    int *ids = (a1 - a0 + 1) <= ID_CAP ? s_ids : g_ids;
    float *sc = (a1 - a0 + 1) <= SC_CAP ? s_sc : g_sc;
    int n = 0;
    if (inc_father) { if (lane == 0) ids[0] = prev; n = 1; }
    float m = -INFINITY;   // running max of the cached scores (lane local)
    const long long t_e = clock64();
    // (16 tiles in flight for hub adjacency was measured: the extra registers spill and the kernel gets slower)
    enumerate_children<U>(d, tb, a0, a1, cached, ids, sc, lane, n, m, stg);
    __syncwarp();
    const long long t_s = clock64();
    cyc[0] += (unsigned int)(t_s - t_e);
    n_out = n; ids_out = ids; sc_out = sc; m_out = m;
    // n == 1: softmax = [1.0], cdf = [1.0], and 1.0 > u for every uniform u in [0, 1): the draw is index 0
    // whatever the score is, so neither the score nor the CDF is computed (leaves of the BFS tree: [father])
    if (n <= 1) return;
    if (!cached || inc_father) {
        if constexpr (CPL == WIDE_CPL) {
            float *s_row = walk_wide_row(s_sc);
            load_row_wide(d.emb, d.ld, cur, s_row, lane);
            score_list_wide(d.emb, d.bias, d.ld, s_row, ids, sc, cached ? 1 : n, cur, lane);
        } else {
            float4 c4[CPL];
            load_row<CPL>(d.emb, d.ld, cur, lane & 7, c4);
            score_list<CPL>(d.emb, d.bias, d.ld, c4, ids, sc, cached ? 1 : n, cur, lane);
        }
        rows_gathered += 1u + (unsigned)(cached ? 1 : n);
    }
    if (cached) {
        m = warp_max(m);
        if (inc_father) m = fmaxf(m, sc[0]);
    } else {
        m = list_max(sc, n, lane);
    }
    m_out = m;
    cyc[1] += (unsigned int)(clock64() - t_s);
}

// warp-aggregated append of `v` for the lanes with `take` (one atomic per warp)
template <class T>
__device__ __forceinline__ void warp_append(bool take, T *list, unsigned *cnt, const T &v, int lane) {
    const unsigned mk = __ballot_sync(FULL, take);
    if (!mk) return;
    const int leader = __ffs(mk) - 1;
    unsigned base = 0;
    if (lane == leader) base = atomicAdd(cnt, (unsigned)__popc(mk));
    base = __shfl_sync(FULL, base, leader);
    if (take) list[base + __popc(mk & ((1u << lane) - 1u))] = v;
}

}  // namespace gg
