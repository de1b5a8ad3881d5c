/*
 * gg_oracle.h -- TEST INFRASTRUCTURE ONLY (tier "T1", the canonical CPU oracle).
 *
 * A plain-C, single-threaded restatement of GraphGAN's graph-softmax walk
 * (reference: src/GraphGAN/graph_gan.py:182-270, src/utils.py:131-133 and the legacy
 * numpy RandomState.choice inverse-CDF step called at graph_gan.py:262) with a FULLY
 * SPECIFIED arithmetic, so that the sm_90a kernels in graphgan_b200/csrc can execute
 * the identical operation sequence and be compared bit-for-bit.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
 * legs may load this library.  The product path never does.
 *
 * Parity status: the reference's TF1.8 kernels cannot run here (no TensorFlow), so the
 * dense arithmetic (sgemm order, numpy SIMD exp) is "parity unpinned"; the control flow,
 * RNG consumption, candidate order and tree mutation ARE pinned against the reference's
 * own Python (tests/golden/make_golden.py imports it from a reference checkout).
 *
 * Canonical arithmetic (shared with the CUDA kernels, see DESIGN.md section 3):
 *   rows      : [N, ld] fp32, ld = round_up(d, 32), zero padded.
 *   dot       : 8 virtual lanes g; lane g owns float4 chunks g, g+8, g+16, ...; one fmaf
 *               chain per lane in (chunk, x,y,z,w) order starting from +0; then butterfly
 *               adds xor 4, 2, 1.
 *   score     : dot + bias[cand]                                   (fp32 add)
 *   softmax   : m = max; e_i = exp_c(s_i - m); tiles of 32 candidates; tile sum = butterfly
 *               adds xor 16,8,4,2,1 over the 32 slots (missing = +0); S = T_0 + T_1 + ...
 *               sequentially; p_i = e_i / S                         (fp32 divide)
 *   cdf       : x_i = (double)p_i; per tile Kogge-Stone inclusive scan (offsets 1,2,4,8,16);
 *               cdf_i = C_t + scan_i with C_0 = 0, C_{t+1} = C_t + scan_31; total = C_last
 *   choice    : first i with (cdf_i / total) > u                   (fp64 divide) == numpy's
 *               cdf /= cdf[-1]; searchsorted(cdf, u, side='right')
 *   exp_c     : Cephes-style range reduction + degree-5 polynomial, explicit fmaf, returns
 *               exactly 0 below -86 (see gg_oracle.c).
 *   uniform   : u = ((a >> 5) * 2^26 + (b >> 6)) / 2^53 from two 32-bit words (same
 *               construction as MT19937 random_sample); words come from Philox4x32-10 with
 *               key = (seed_lo, seed_hi), counter = (root, walk, step, pass_tag), or from a
 *               caller supplied stream of doubles consumed in reference order.
 */
#ifndef GG_ORACLE_H
#define GG_ORACLE_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum { GGO_NOTRUN = 0, GGO_DONE = 1, GGO_VOID = 2, GGO_SKIPPED = 3 };
enum { GGO_RNG_PHILOX = 0, GGO_RNG_STREAM = 1 };

void ggo_philox4x32_10(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4]);
double ggo_u53(uint32_t a, uint32_t b);
float ggo_exp(float x);
float ggo_dot(const float *a, const float *b, int ld);

/* softmax + inverse-CDF choice over n scores (overwrites sc with e_i). returns index. */
int ggo_choose(float *sc, int n, double u);

/* BFS parent array in the reference's discovery order (graph_gan.py:84-108):
 * parent[root] = -1, unreachable = -1. queue: scratch of n int32. returns #reached. */
int64_t ggo_bfs_parent(int64_t n, const int64_t *indptr, const int32_t *adj, int32_t root,
                       int32_t *parent, int32_t *queue);

typedef struct {
    int64_t n_node;
    int32_t ld;
    const float *emb;        /* [N, ld] generator embedding_matrix  */
    const float *bias;       /* [N]     generator bias_vector        */
    const int64_t *indptr;   /* [N+1]   unique-neighbour CSR, first-occurrence file order */
    const int32_t *adj;
    int64_t n_roots;
    const int32_t *roots;    /* [R] node ids, processed in this order */
    const int32_t *parent;   /* [R, N] */
    const int64_t *walk_ptr; /* [R+1] prefix sum of per-root sample_num */
    int32_t for_d;
    uint32_t *d1_bits;       /* "father removed" bitset over CSR edge index; D writes, G reads */
    int32_t rng_mode;
    uint64_t seed;
    uint32_t pass_tag;
    const double *stream;    /* GGO_RNG_STREAM: doubles consumed in reference order */
    int64_t n_stream;
    double update_ratio;
    int32_t max_path;        /* paths row stride (0 = do not record) */
    /* outputs */
    int32_t *samples;        /* [W] */
    int32_t *status;         /* [W] */
    int32_t *first_edge;     /* [W] CSR edge index of the depth-1 node chosen at the root step */
    int32_t *wsteps;         /* [W] */
    int32_t *wsuml;          /* [W] */
    int32_t *paths;          /* [W, max_path] */
    int32_t *path_len;       /* [W] */
    int32_t *root_ok;        /* [R] 1 = accepted (reference: "neg is not None") */
    int64_t *counters;       /* [8]: steps, sumL, stream consumed, path overflow, max |L|, ... */
} ggo_walk_args;

int ggo_walk_pass(const ggo_walk_args *a);

#ifdef __cplusplus
}
#endif
#endif
