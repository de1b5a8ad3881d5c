/*
 * graphgan_b200.h -- C ABI of libgraphgan_b200.so, the H100 (sm_90a) implementation of
 * GraphGAN's scoring-and-sampling hot path.
 *
 * The reference (hwwang55/GraphGAN) has no native code and no FFI: its seam is the five
 * tf.Session.run(fetch, feed_dict) call sites of src/GraphGAN/graph_gan.py (154, 173, 220,
 * 238, 298).  Each entry point below states the reference code it replaces; the Python
 * binding a maintainer adds is shown in INTEGRATION.md (ctypes, graphgan_b200/_cabi.py).
 *
 * Conventions
 *   - every pointer marked "device" is a CUDA device pointer owned by the caller (in the
 *     Python host: torch tensors used only as memory containers, passed as data_ptr()).
 *   - `stream` is a cudaStream_t passed as void*; all work is asynchronous on it, no hidden
 *     synchronisation, no allocation.  Scratch is caller supplied (query *_scratch_bytes).
 *   - return 0 on success, non-zero on CUDA / argument error; gg_last_error() gives the
 *     message for the calling thread.  Nothing aborts.
 *   - embedding rows are fp32 [N, ld], zero padded, with ld = 32, 64, 128, 256 or 512 (the smallest that holds
 *     n_emb, so n_emb <= 512): every entry point that takes ld rejects other values.
 *   - graph = two CSRs in the reference's adjacency-file order (src/utils.py:27-37):
 *       raw  : graph[i] as read (duplicates and self-loops kept) -> positives, sample_num
 *       walk : first occurrences only, self-loops dropped        -> BFS trees and walks
 */
#ifndef GRAPHGAN_B200_H
#define GRAPHGAN_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GG_ABI_VERSION 11  /* 11: gg_adam_apply_dense, then gg_expected_g_grad, then gg_generator_dist_d and
                              gg_expected_d_grad, then gg_best_response, gg_best_response_grad and gg_best_response_spmm,
                              then gg_expected_g_moments
                              (additions: every older entry point keeps
                              its signature and meaning, and _cabi.lib() refuses a library that lacks a declared symbol); 10: gg_game_value_grad_d; 9: gg_game_value_grad; 8: gg_game_value; 7: gg_generator_dist */

/* walk status codes (per walk) */
enum { GG_NOTRUN = 0, GG_DONE = 1, GG_VOID = 2, GG_SKIPPED = 3 };
/* rng modes */
enum {
    GG_RNG_PHILOX = 0, /* Philox4x32-10, key=(seed), counter=(root, walk, step, pass_tag): order free */
    GG_RNG_STREAM = 1  /* caller supplied doubles consumed in the reference's sequential order
                          (np.random.rand at graph_gan.py:189/209, np.random.choice at :262) */
};
/* counters[] slots written by gg_walk_finalize (reference semantics: walks after a root's
 * first voiding walk do not exist) */
enum {
    GG_CNT_STEPS = 0, GG_CNT_SUML = 1, GG_CNT_ACCEPTED = 2, GG_CNT_OK_ROOTS = 3,
    GG_CNT_PATH_OVERFLOW = 4, GG_CNT_RAW_STEPS = 5, GG_CNT_RAW_SUML = 6, GG_CNT_STREAM_USED = 7,
    GG_CNT_ROWS_GATHERED = 8, /* embedding rows the walk kernel actually fetched (on-demand scores + cur rows) */
    /* warp-cycles (clock64, summed over warps) spent per phase of the walk kernel */
    GG_CNT_CYC_ENUM = 9, GG_CNT_CYC_SCORE = 10, GG_CNT_CYC_CHOOSE = 11, GG_CNT_CYC_STEP0 = 12,
    GG_CNT_CYC_STEP1 = 13, GG_CNT_CYC_STEP2P = 14, GG_CNT_CYC_WALK = 15,
    GG_CNT_SLOTS = 16
};

const char *gg_last_error(void);
int gg_abi_version(void);

/* ------------------------------------------------------------------------------------------
 * K1: graph-softmax walk.  Replaces GraphGAN.sample (graph_gan.py:225-270) together with the
 * generator.all_score fetch at :238 (scores are computed on demand for the candidates only,
 * generator.py:21), utils.softmax (utils.py:131-133) and np.random.choice's inverse-CDF
 * draw (:262), for a whole batch of roots at once.
 * ------------------------------------------------------------------------------------------ */
typedef struct gg_walk_desc {
    int64_t n_node;
    int32_t ld;                 /* row stride in floats: 32, 64, 128, 256 or 512 (see Conventions) */
    const float *emb;           /* device [N, ld]  generator.embedding_matrix (generator.py:11-14) */
    const float *bias;          /* device [N]      generator.bias_vector      (generator.py:15)    */
    const int64_t *indptr;      /* device [N+1]    walk CSR */
    const int32_t *adj;         /* device [nnz]    */
    int64_t n_roots;
    const int32_t *roots;       /* device [R] root node ids (batch order = reference root order) */
    const uint32_t *tree_bits;  /* device [R, tree_words] BFS trees (gg_bfs_build): bit e of row k is set iff adj[e]
                                   is a child of entry e's source node in the tree of roots[k] */
    int64_t tree_words;         /* row stride of tree_bits in 32-bit words (gg_tree_words(nnz)) */
    const int64_t *walk_ptr;    /* device [R+1] exclusive prefix of per-root sample_num */
    int64_t n_walks;            /* = walk_ptr[R] */
    int32_t for_d;              /* graph_gan.py:225 `for_d` */
    int32_t rng_mode;
    uint32_t *d1_bits;          /* device bitset over walk-CSR entries: "father entry removed"
                                   (the in-place tree mutation of graph_gan.py:258-259).
                                   G mode reads it here; D mode sets it in gg_walk_finalize */
    uint64_t seed;
    uint32_t pass_tag;
    int32_t max_path;           /* row stride of paths (0: paths not recorded) */
    const double *stream;       /* device, GG_RNG_STREAM only */
    int64_t n_stream;
    double update_ratio;        /* config.update_ratio (graph_gan.py:189/209) */
    int32_t max_cand;           /* >= max walk-CSR degree + 1 */
    int32_t phase_mask;         /* 0 = whole call; 1 = only the depth-1 precompute (root steps + per-pair CDFs), 2 = only
                                   the walk kernel -- lets a profiler time the two stages of one pass separately */
    /* per-walk outputs, device [W] */
    int32_t *samples;           /* sampled node (graph_gan.py:265) or -1 */
    int32_t *status;
    int32_t *first_edge;        /* walk-CSR entry of the depth-1 node chosen at the root step */
    int32_t *wsteps;            /* choices made */
    int32_t *wsuml;             /* sum of candidate-list lengths */
    int32_t *paths;             /* device [W, max_path] or NULL */
    int32_t *path_len;          /* device [W] or NULL */
    unsigned long long *counters; /* device [GG_CNT_SLOTS] */
    void *scratch;              /* device, gg_walk_scratch_bytes(max_cand) */
    int64_t scratch_bytes;
    unsigned int *work_counter; /* device, 1 word, zeroed by the call */
    /* optional per-pass precomputation (identical results, far less traffic; see DESIGN.md section 5) */
    const float *edge_score;    /* device [nnz] all_score[u, adj[e]] for walk-CSR entries of nodes with
                                   degree >= hub_threshold (gg_hub_scores); NULL = always score on demand */
    const double *root_q;       /* device: per root, the normalised CDF of its root step (gg_root_cdf);
                                   NULL = compute the root step per walk */
    const int64_t *rq_ptr;      /* device [R+1] offsets into root_q (prefix of the roots' walk-CSR degrees) */
    int32_t hub_threshold;
    int32_t no_tma;             /* 1 = enumerate hub lists with plain loads instead of cp.async.bulk staging (A/B measurement;
                                   identical results) */
    const int32_t *walk_slot;   /* optional device [W]: root slot of every walk (saves a binary search per walk) */
    /* optional depth-1 reuse (GG_RNG_PHILOX, needs root_q + walk_slot): the walks of a root that pick the same
       depth-1 child share one candidate list.  gg_walk_sample first runs the root step of every walk and counts
       the walks per (root, child) pair, builds the candidate ids and the un-normalised canonical CDF (plus its
       total) of every pair picked by at least two walks, and the walk kernel then only inverts it (pairs picked
       once are handled inside their walk).  Indexing: pair (root slot k, i-th neighbour) <-> pos = rq_ptr[k] + i,
       pos < s1_nq. */
    int64_t s1_nq;              /* = rq_ptr[R] */
    const int32_t *s1_slot;     /* device [s1_nq] root slot of every pair */
    const int64_t *s1_ptr;      /* device [s1_nq+1] exclusive prefix of (degree(child) + 1): pool offsets */
    int32_t *s1_cnt;            /* device [s1_nq] scratch: walks per pair */
    int32_t *s1_n;              /* device [s1_nq] out: list length of a pair (0 = void) */
    double *s1_q;               /* device pool [s1_ptr[s1_nq]]: per pair c[0..n-1] = carry + scan(e/S), c[n] = total */
    int32_t *s1_ids;            /* device pool: candidate ids */
    int32_t *first_idx;         /* device [W] scratch: root-step choice of every walk */
    const int32_t *s1_order;    /* optional device [s1_nq]: the (root, child) pairs sorted by decreasing child degree; with it
                                 * step1_cdf_kernel pulls pairs from a queue (largest lists first) instead of striding */
    const int32_t *walk_order;  /* optional device [W]: the order in which walk_kernel starts the walks (a permutation of
                                 * 0..W-1, e.g. expensive roots first); results do not depend on it (Philox mode) */
    /* optional level-synchronous steps (needs the depth-1 reuse): all unfinished walks take step s together -- one
       kernel enumerates the candidate lists, one gathers the candidates' rows and draws -- for steps 1..flat_steps;
       the persistent kernel finishes the walks that are still alive after that.  On the levels the library shares
       (step 2 by default) the walks of a root that stand on the same node draw from one candidate list and CDF,
       keyed by (root slot, node): n_node must be set.  Identical results. */
    void *flat_buf;             /* device scratch of gg_walk_flat_bytes(n_walks, hub_threshold, flat_steps) bytes */
    int64_t flat_bytes;
    int32_t flat_steps;         /* 0 = off (persistent kernel only); <= 14 */
    int32_t flat_reserved;
} gg_walk_desc;

/* all_score[u, v] = e_u.e_v + b_v (generator.py:21) for the listed walk-CSR entries e = (u -> v), grouped by
 * target: pairs = device int32 [n_pairs, 2] of (u, e), items = device int32 [n_items, 4] of (v, first, count, unused),
 * item t covering pairs[first, first + count), all of them entries into v; edge_score[e] is written for every listed
 * pair.  Must be re-run whenever the generator's embeddings change (i.e. once per sampling pass). */
int gg_hub_scores(int64_t n_items, const int32_t *items, const int32_t *pairs, const float *emb, const float *bias,
                  int32_t ld, float *edge_score, void *stream);
/* Root-step softmax + CDF, once per root per pass: root_q[rq_ptr[k] + i] = cdf_i / cdf_last over the
 * candidates tree[root][1:] (graph_gan.py:250,260-262).  Uses d->{roots, n_roots, indptr, adj, emb, bias,
 * ld, rq_ptr, edge_score, hub_threshold}.  root_sc: device float scratch of rq_ptr[R] entries. */
int gg_root_cdf(const gg_walk_desc *d, float *root_sc, double *root_q, void *stream);

int gg_walk_scratch_bytes(int32_t max_cand, int64_t *bytes);
int gg_walk_flat_bytes(int64_t n_walks, int32_t hub_threshold, int32_t flat_steps, int64_t *bytes);
int gg_walk_sample(const gg_walk_desc *d, void *stream);

/* Per root: find the first voiding walk (graph_gan.py:252-257 returns None for the WHOLE
 * root), blank the walks after it, set root_ok ("neg is not None and len(pos) != 0",
 * graph_gan.py:192), apply the father-removal bits of the surviving D walks, and reduce the
 * counters. */
int gg_walk_finalize(int64_t n_roots, const int64_t *walk_ptr, int32_t for_d, int32_t *samples,
                     int32_t *status, const int32_t *first_edge, int32_t *wsteps, int32_t *wsuml,
                     int32_t *path_len, uint32_t *d1_bits, int32_t *root_ok,
                     unsigned long long *counters, void *stream);

/* The exact generator distribution G(v | root) (csrc/gdist.cu, DESIGN.md section 5.1): for every root k of the batch,
 * dist[k, v] = the probability that one G-mode walk from roots[k] (graph_gan.py:225-270, for_d = 0) stops at v, computed
 * from the walk's own candidate lists and canonical CDFs in fp64 -- not sampled.  Step law of a list with canonical CDF q:
 * pi(x_j) = (ceil(q_j 2^53) - ceil(q_{j-1} 2^53)) / 2^53; reach(root) = 1, reach(child) = reach(a) * pi_a(child),
 * dist[k, v] = reach(v) * pi_v(father(v)), each one fixed chain of fp64 products (bit-reproducible).  dist[k, root] = 0 and
 * dist = 0 off the tree.  root_ok[k] = 1 when the walks of the root cannot void (the root has children, and no reachable
 * depth-1 node whose father entry is removed has an empty list); root_ok[k] = 0 rows are all zero.
 * Uses d->{n_node, ld, emb, bias, indptr, adj, n_roots, roots, tree_bits, tree_words, d1_bits (NULL: no father entry
 * removed), edge_score + hub_threshold (optional: cached scores of nodes with degree >= hub_threshold, gg_hub_scores; the
 * same bits either way)} and adds the embedding rows it fetches to d->counters[GG_CNT_ROWS_GATHERED] when counters is set;
 * the walk fields are ignored.  dist: device fp64 [n_roots, n_node]; root_ok: device [n_roots]; n_roots * n_node < 2^31.
 * scratch: device, at least gg_generator_dist_scratch_bytes(n_node, nnz, n_roots) bytes (host-only size computation;
 * O(n_roots * (nnz + n_node))).  One cooperative launch. */
int gg_generator_dist_scratch_bytes(int64_t n_node, int64_t nnz, int64_t n_roots, int64_t *bytes);
int gg_generator_dist(const gg_walk_desc *d, double *dist, int32_t *root_ok, void *scratch, int64_t scratch_bytes,
                      void *stream);

/* The D-mode walk law (csrc/gdist.cu, DESIGN.md section 5.7): gg_generator_dist for the walks of a discriminator pass
 * (graph_gan.py:225-270, for_d = 1).  The root's list is its children, every depth-1 node's list its children (the root
 * is removed whatever d->d1_bits holds, so d1_bits is not read and may be NULL), a deeper node's list [father] +
 * children.  dist[k, v] = reach(v) * pi_v(father(v)) for depth >= 2, 0 at the root and at depth 1.  p_void[k] (device
 * fp64 [n_roots]) = the sum of reach(a) over the depth-1 leaves a: the probability that one D walk voids the root's pass
 * (graph_gan.py:255-257); a sum of multiples of 2^-53 at most 1, exact in any order.  root_ok[k] = 1 iff the root has
 * children.  Every other field, the scratch (gg_generator_dist_scratch_bytes) and the limits as for gg_generator_dist. */
int gg_generator_dist_d(const gg_walk_desc *d, double *dist, double *p_void, int32_t *root_ok, void *scratch,
                        int64_t scratch_bytes, void *stream);

/* The GraphGAN game value per root, exactly (csrc/value.cu, DESIGN.md section 5.2; Wang et al., AAAI-18, Eq. 1):
 *   V_c = pos_c + neg_c,  pos_c = -(1 / |graph[c]|) sum_k bce(s(c, graph[c][k]), 1)  (raw CSR, entry order, duplicates and
 *   self-loops count),  neg_c = -sum_v dist[k, v] bce(s(c, v), 0)  (v with dist[k, v] = 0 contribute exactly 0),
 * for c = roots[k], with the discriminator's score s(c, v) = fp32 canonical dot(emb[c], emb[v]) + bias[v] (the bits of
 * gg_pair_reward's score before its clip) and bce(s, y) = (max(s, 0) - s y) + log1p(exp(-|s|)) in fp64
 * (sigmoid_cross_entropy_with_logits, discriminator.py:26-30).  dist / root_ok: gg_generator_dist's outputs for the same
 * roots (the generator's G-mode law).  ok[k] = 1 iff |graph[c]| > 0 and root_ok[k] == 1; otherwise pos[k] = neg[k] = 0.
 * Every sum runs in a fixed order: the bits depend on the inputs only, not on the number or order of the roots.
 * emb: device [n_node, ld] (the discriminator's rows), bias: device [n_node]; raw_indptr / raw_adj: device raw CSR;
 * roots: device [n_roots]; dist: device fp64 [n_roots, n_node]; root_ok: device [n_roots]; pos, neg: device fp64
 * [n_roots]; ok: device [n_roots].  scratch: device, at least gg_game_value_scratch_bytes(n_node, n_roots) bytes
 * (host-only size computation, 8 bytes per root and 512 nodes).  Two launches. */
int gg_game_value_scratch_bytes(int64_t n_node, int64_t n_roots, int64_t *bytes);
int gg_game_value(int64_t n_node, int32_t ld, const float *emb, const float *bias, const int64_t *raw_indptr,
                  const int32_t *raw_adj, int64_t n_roots, const int32_t *roots, const double *dist,
                  const int32_t *root_ok, double *pos, double *neg, int32_t *ok, void *scratch, int64_t scratch_bytes,
                  void *stream);

/* The exact generator gradient of the game value (csrc/value_grad.cu, DESIGN.md section 5.3): for the roots of g (the
 * generator's law as gg_generator_dist computes it from g's fields) and the discriminator d_emb / d_bias, writes pos, neg
 * and ok with the bits of gg_game_value and ADDS the gradient of sum_{ok c} V_c with respect to the generator's padded rows
 * (g->emb, ld columns) and biases into grad_emb (device fp64 [n_node, ld]) and grad_bias (device fp64 [n_node]):
 *   grad_G V_c = -sum over lists a, candidates x of w_a(x) grad s(a, x),  w_a(x) = F_a(x) - pi_a(x) T(a),
 * T(a) = the sum of h(u) = G(u | c) bce(s_D(c, u), 0) over the subtree of a, F_a(x) = T(x) for a child, h(a) for the father.
 * Pad columns receive exactly 0.  Each node's row takes the roots in the order given as one fp64 chain per coordinate,
 * continued from the value already in grad_emb / grad_bias: pass the roots in ascending id order (and chunks in order)
 * for bits that do not depend on the order or the chunking.  d_emb has g->ld columns.  Other arguments as for
 * gg_generator_dist and gg_game_value.  scratch: device, at least gg_game_value_grad_scratch_bytes(n_node, nnz, n_roots)
 * bytes (host-only size computation; gg_generator_dist's plus 28 bytes per (root, node)). */
int gg_game_value_grad_scratch_bytes(int64_t n_node, int64_t nnz, int64_t n_roots, int64_t *bytes);
int gg_game_value_grad(const gg_walk_desc *g, const float *d_emb, const float *d_bias, const int64_t *raw_indptr,
                       const int32_t *raw_adj, double *pos, double *neg, int32_t *ok, double *grad_emb, double *grad_bias,
                       void *scratch, int64_t scratch_bytes, void *stream);

/* The exact discriminator gradient of the game value (csrc/value_dgrad.cu, DESIGN.md section 5.4): for the roots, dist and
 * root_ok of gg_game_value (the other arguments as there), ADDS the gradient of sum_{ok c} V_c with respect to the
 * discriminator's padded rows (emb, ld columns) and biases into grad_emb (device fp64 [n_node, ld]) and grad_bias (device
 * fp64 [n_node]):
 *   W[k, v] = dV_c / ds(c, v) = n_kv sigma(-s) / |graph[c]| - dist[k, v] sigma(s)   (c = roots[k], s the canonical fp32
 *   score of gg_game_value, sigma in fp64; n_kv the count of v in the raw list graph[c], duplicates and self-loops too),
 *   grad_bias[v] += W[k, v],  grad_emb[v] += W[k, v] emb[c],  grad_emb[c] += sum_v W[k, v] emb[v]
 * for ok[k] = 1 only (the ok of gg_game_value); lambda_dis is not included.  Pad columns receive exactly 0.  Each node's
 * row takes the roots in the order given as one fp64 chain per coordinate, continued from the value already in grad_emb /
 * grad_bias: pass the roots in ascending id order (and chunks in order) for bits that do not depend on the order or the
 * chunking.  scratch: device, at least gg_game_value_grad_d_scratch_bytes(n_node, ld, n_roots) bytes (host-only size
 * computation; 12 bytes per (root, node) plus 8 ld bytes per root and 2048 nodes).  Five launches and one memset. */
int gg_game_value_grad_d_scratch_bytes(int64_t n_node, int32_t ld, int64_t n_roots, int64_t *bytes);
int gg_game_value_grad_d(int64_t n_node, int32_t ld, const float *emb, const float *bias, const int64_t *raw_indptr,
                         const int32_t *raw_adj, int64_t n_roots, const int32_t *roots, const double *dist,
                         const int32_t *root_ok, double *grad_emb, double *grad_bias, void *scratch, int64_t scratch_bytes,
                         void *stream);

/* The exact expectation of the reference's discriminator step of one pass (csrc/value_dgrad.cu, DESIGN.md section 5.7):
 * for the roots and the D-mode law of gg_generator_dist_d (dist_d, p_void, root_ok) and the discriminator emb / bias
 * (other arguments as for gg_game_value_grad_d), writes accept (device fp64 [n_roots]): P_acc = (1 - p_void)^deg_c,
 * deg_c = |graph[c]|, by square-and-multiply from the least significant bit (one fp64 product per step), 0 unless
 * deg_c > 0 and root_ok = 1; ok_ref = accept > 0.  ADDS the expectation of -grad sum_rows bce over the rows
 * prepare_data_for_d emits for the root (deg_c positives from the raw list, deg_c negatives from Q = dist_d / (1 - p_void),
 * emitted with probability P_acc) into grad_emb / grad_bias with the assembly of gg_game_value_grad_d, W replaced by
 *   W_ref[k, v] = fl(fl(deg_c P_acc) dgrad_w(n_kv, deg_c, Q[k, v], s))   (dgrad_w: gg_game_value_grad_d's W per pair)
 * for ok_ref = 1 only; lambda_dis, the 1 / batch mean and update_ratio are not included.  The same order contract as
 * gg_game_value_grad_d.  scratch: device, at least gg_expected_d_grad_scratch_bytes(n_node, ld, n_roots) bytes (host-only
 * size computation; gg_game_value_grad_d_scratch_bytes' plus 4 bytes per root).  Six launches and one memset. */
int gg_expected_d_grad_scratch_bytes(int64_t n_node, int32_t ld, int64_t n_roots, int64_t *bytes);
int gg_expected_d_grad(int64_t n_node, int32_t ld, const float *emb, const float *bias, const int64_t *raw_indptr,
                       const int32_t *raw_adj, int64_t n_roots, const int32_t *roots, const double *dist_d,
                       const double *p_void, const int32_t *root_ok, double *accept, double *grad_emb, double *grad_bias,
                       void *scratch, int64_t scratch_bytes, void *stream);

/* The game value against the best discriminator (csrc/best_response.cu, DESIGN.md section 5.8): for the roots of g (the
 * generator's G-mode law as gg_generator_dist computes it from g's fields, current father-removal bits), with
 * p(a) = mult[e] / |graph[c]| for the walk-CSR entry e = (c -> a) and G(a) = fl(pi_c(a) pi_a(c)) (the bits of
 * gg_generator_dist's dist[k, a]) at the depth-1 nodes a:
 *   vstar[k] = -sum_a (p(a) log1p(G(a) / p(a)) + G(a) log1p(p(a) / G(a)))  (= max_D V_c(G, D) = 2 JSD(p || G) - log 4;
 *              the G term is 0 where G(a) = 0),  hit[k] = sum_a G(a),
 * both summed over c's walk-CSR entries in the order of DESIGN.md section 5.8.  ok[k] = 1 iff |graph[c]| > 0 and
 * gg_generator_dist's root_ok is 1 (the bits of gg_game_value's ok); otherwise vstar[k] = hit[k] = 0.  raw_indptr: the raw
 * CSR's [n_node + 1]; mult: device int32 [nnz], mult[e] = the count of adj[e] in the raw list of e's row.  Only the
 * depth-1 lists are built.  scratch: device, at least gg_best_response_scratch_bytes(n_node, nnz, n_roots) bytes
 * (host-only size computation; O(n_roots * (nnz + n_node))); n_roots * n_node < 2^31.  One cooperative launch. */
int gg_best_response_scratch_bytes(int64_t n_node, int64_t nnz, int64_t n_roots, int64_t *bytes);
int gg_best_response(const gg_walk_desc *g, const int64_t *raw_indptr, const int32_t *mult, double *vstar, double *hit,
                     int32_t *ok, void *scratch, int64_t scratch_bytes, void *stream);
/* gg_best_response, and the gradient of sum_{ok c} vstar_c with respect to g's rows and biases as per-entry coefficients
 * ADDED to the caller's accumulators acc_coef and acc_bias (device fp64 [nnz]): the edge coefficient c_e on both entries of
 * each tree edge, the bias coefficient on the receiving node's entry.  The roots are taken in the order given, each entry
 * one fp64 chain: pass the roots in ascending id order (and chunks in order) for bits that do not depend on the order or
 * the chunking.  rev: gg_reverse_entries' (a symmetric walk CSR).  gg_best_response_spmm turns the accumulators into the
 * gradient.  scratch: gg_best_response_grad_scratch_bytes(n_node, nnz, n_roots) bytes (20 bytes per (root, node) more than
 * gg_best_response's).  One cooperative launch with one grid barrier per ok root. */
int gg_best_response_grad_scratch_bytes(int64_t n_node, int64_t nnz, int64_t n_roots, int64_t *bytes);
int gg_best_response_grad(const gg_walk_desc *g, const int64_t *raw_indptr, const int32_t *mult, const int32_t *rev,
                          double *vstar, double *hit, int32_t *ok, double *acc_coef, double *acc_bias, void *scratch,
                          int64_t scratch_bytes, void *stream);
/* The gradient from gg_best_response_grad's accumulators, ADDED to grad_emb (device fp64 [n_node, ld]) and grad_bias
 * (device fp64 [n_node]): row y, coordinate i, is one fp64 chain over y's walk-CSR entries e in entry order,
 * acc = fma(-acc_coef[e], emb[adj[e]][i], acc), and the bias accb = accb - acc_bias[e] (zero coefficients skipped).  Pad
 * columns stay exactly 0.  No scratch.  One launch. */
int gg_best_response_spmm(int64_t n_node, int32_t ld, const int64_t *indptr, const int32_t *adj, const float *emb,
                          const double *acc_coef, const double *acc_bias, double *grad_emb, double *grad_bias, void *stream);

/* The exact expectation of the reference's generator step (csrc/value_gref.cu, DESIGN.md section 5.6): for the roots of g
 * (the generator's law as gg_generator_dist computes it from g's fields, G mode, current father-removal bits) and the
 * discriminator d_emb / d_bias (g->ld columns), writes root_ok (device int32 [n_roots], the root_ok of gg_generator_dist)
 * and n_pairs (device fp64 [n_roots]: the expected number of window pairs per walk, sum_y reach(y) 2 min(window, depth(y)),
 * 0 where root_ok = 0), and ADDS the expected per-walk sum of the production pair gradients of the window pairs
 * (graph_gan.py:204-223 and :272-291 with config.window_size = window, generator.py:22-31) into grad_emb (device fp64
 * [n_node, ld]) and grad_bias (device fp64 [n_node]):
 *   for every reached y != root, d = 1 .. min(window, depth(y)), x = anc_d(y), and both ordered pairs (n1, n2) of {x, y}:
 *   grad_emb[n1] += rho kappa emb[n2],  grad_emb[n2] += rho kappa emb[n1],  grad_bias[n2] += rho kappa
 * rho = reach(y), the probability that a walk passes y; kappa = the fp32 coefficient of gg_pair_grad mode 1 with batch_total
 * 1 and the reward of gg_pair_reward as a_k (lambda_gen and the 1 / batch mean are not included).  The sampled pairs are
 * held fixed: no term flows through the law.  Pad columns receive exactly 0.  window: 1 .. 8.  Each node's row takes the
 * roots in the order given as one fp64 chain per coordinate, continued from the value already in grad_emb / grad_bias:
 * pass the roots in ascending id order (and chunks in order) for bits that do not depend on the order or the chunking.
 * scratch: device, at least gg_expected_g_grad_scratch_bytes(n_node, nnz, n_roots, window) bytes (host-only size
 * computation; gg_generator_dist's plus 20 + 8 window bytes per (root, node)). */
int gg_expected_g_grad_scratch_bytes(int64_t n_node, int64_t nnz, int64_t n_roots, int32_t window, int64_t *bytes);
int gg_expected_g_grad(const gg_walk_desc *g, const float *d_emb, const float *d_bias, int32_t window, double *n_pairs,
                       int32_t *root_ok, double *grad_emb, double *grad_bias, void *scratch, int64_t scratch_bytes,
                       void *stream);
/* gg_expected_g_grad, and the second moment of one walk's step (csrc/value_gref.cu, DESIGN.md section 5.9).  A G walk
 * that stops at y adds a fixed vector s(y), the window-pair gradient of the body root -> y; P(y) is gg_generator_dist's
 * law.  Writes, per root, sq = sum_y P(y) |s(y)|^2 and mn = |m|^2 (device fp64 [n_roots]; 0 where root_ok = 0), m the
 * root's expected step (its contribution to grad_emb / grad_bias); the norms run over the rows and the biases.  sq - mn
 * is the trace of the covariance of one walk's step.  sq_node (device fp64 [n_roots, n_node], or NULL): |s(y)|^2 per
 * node, 0 at the root and at nodes not reached.  n_pairs, root_ok, grad_emb and grad_bias are gg_expected_g_grad's, bit
 * for bit, and the arguments are checked as there.  The bits depend on the inputs only.  scratch: device, at least
 * gg_expected_g_moments_scratch_bytes(n_node, nnz, n_roots, window) bytes (host-only size computation;
 * gg_expected_g_grad's plus 16 bytes per (root, node)). */
int gg_expected_g_moments_scratch_bytes(int64_t n_node, int64_t nnz, int64_t n_roots, int32_t window, int64_t *bytes);
int gg_expected_g_moments(const gg_walk_desc *g, const float *d_emb, const float *d_bias, int32_t window, double *n_pairs,
                          int32_t *root_ok, double *sq, double *mn, double *sq_node, double *grad_emb, double *grad_bias,
                          void *scratch, int64_t scratch_bytes, void *stream);

/* prepare_data_for_d's output rows (graph_gan.py:192-201): for every accepted root, in batch
 * order: [i]*k + [i]*k | pos + neg | 1*k + 0*k.  row_ptr: device [R+1] scratch/out (exclusive
 * scan of 2*len(pos) over accepted roots); n_rows_out: device int64. */
int gg_emit_d_rows(int64_t n_roots, const int32_t *roots, const int64_t *walk_ptr,
                   const int64_t *pos_indptr, const int32_t *pos_flat, const int32_t *root_ok,
                   const int32_t *samples, int64_t *row_ptr, int32_t *center, int32_t *neighbor,
                   int32_t *label, int64_t *n_rows_out, void *stream);

/* ------------------------------------------------------------------------------------------
 * Tree construction: GraphGAN.construct_trees (graph_gan.py:84-108) for a batch of roots.  A tree is one bit per
 * walk-CSR entry: bit e of row k is set iff adj[e] is a child of the source node of entry e in the tree of
 * roots[k] (first discoverer in the reference's FIFO / adjacency order).  tree_bits: device [R, tree_words],
 * tree_words = gg_tree_words(nnz) (= ceil(nnz / 32) + 1); rows are zeroed by the call.  The walk never needs a
 * father pointer (it only descends: the father is the previous node); gg_tree_parent expands rows into the
 * parent-array form (parent[root] = parent[unreachable] = -1) for tests and host-side consumers.
 * ------------------------------------------------------------------------------------------ */
int gg_tree_words(int64_t nnz, int64_t *words);
int gg_bfs_scratch_bytes(int64_t n_node, int64_t nnz, int64_t *bytes);
int gg_bfs_build(int64_t n_node, int64_t nnz, const int64_t *indptr, const int32_t *adj, int64_t n_roots,
                 const int32_t *roots, uint32_t *tree_bits, int64_t tree_words, void *scratch,
                 int64_t scratch_bytes, void *stream);
/* Direction-optimising form.  rev (device [nnz], gg_reverse_entries; static per graph) maps the entry (u -> v) to the
 * entry (v -> u) and lets a level run bottom-up: every undiscovered node picks the visited neighbour with the smallest
 * queue position, the tree row then yields the new nodes in FIFO order (csrc/bfs.cu).  A level runs bottom-up when
 * (adjacency entries of the undiscovered nodes + 4 * frontier nodes) < bottom_up_ratio * (adjacency entries of the
 * frontier); bottom_up_ratio < 0: library default, 0: never.  rev == NULL: plain gg_bfs_build.  The trees are the
 * same bit for bit in every mode.  gg_reverse_entries sets *n_missing (device) to the number of entries without a
 * reverse (rev = -1 there): a CSR with n_missing != 0 is not symmetric and must be built with rev == NULL. */
#define GG_BFS_NO_SORTED_BOTTOM_UP 1   /* flags: disable the small sort-based bottom-up levels (tests / A-B) */
int gg_reverse_entries(int64_t n_node, int64_t nnz, const int64_t *indptr, const int32_t *adj, int32_t *rev,
                       int32_t *n_missing, void *stream);
int gg_bfs_build_ex(int64_t n_node, int64_t nnz, const int64_t *indptr, const int32_t *adj, const int32_t *rev,
                    int64_t n_roots, const int32_t *roots, uint32_t *tree_bits, int64_t tree_words, void *scratch,
                    int64_t scratch_bytes, float bottom_up_ratio, int32_t flags, void *stream);
int gg_tree_parent(int64_t n_node, const int64_t *indptr, const int32_t *adj, int64_t n_roots,
                   const int32_t *roots, const uint32_t *tree_bits, int64_t tree_words, int32_t *parent,
                   void *stream);

/* ------------------------------------------------------------------------------------------
 * K2: pair scoring.  score_k = e_{i_k}.e_{j_k} + b_{j_k} (discriminator.py:21-24 /
 * generator.py:22-25).
 * ------------------------------------------------------------------------------------------ */
/* discriminator.reward (discriminator.py:33-34): log(1 + exp(clip(score, -10, 10))) */
int gg_pair_reward(int64_t n_pairs, const int32_t *node_id, const int32_t *node_neighbor_id,
                   const float *emb, const float *bias, int32_t ld, float *reward, void *stream);
/* generator.all_score rows (generator.py:21) for small N only (tests / source compat) */
int gg_all_score(int64_t n_node, const float *emb, const float *bias, int32_t ld, float *out,
                 void *stream);

/* Sparse gradient of one mini-batch (<= GG_MAX_BATCH pairs), duplicates summed in pair order
 * (TF1.8 AdamOptimizer._apply_sparse_duplicate_indices: unique + segment_sum):
 *   mode 0 = discriminator loss (discriminator.py:26-30), aux = label
 *   mode 1 = generator loss     (generator.py:26-29),     aux = reward
 * outputs: n_unique (device int32), uniq_ids[2B], grad_rows[2B, ld], grad_bias[2B],
 * row_slot: device [N] int32 map, must be all -1 on entry; set for touched rows.
 * batch_total: size of the whole mini-batch when n_pairs is one rank's slice of it (the generator
 * loss is a MEAN over the batch, generator.py:28); 0 = n_pairs. */
#define GG_MAX_BATCH 1024
int gg_pair_grad(int32_t mode, int32_t n_pairs, int32_t batch_total, const int32_t *node_id,
                 const int32_t *node_neighbor_id, const float *aux, const float *emb,
                 const float *bias, int32_t ld, float lambda, int32_t *n_unique, int32_t *uniq_ids,
                 float *grad_rows, float *grad_bias, int32_t *row_slot, void *stream);

/* The same gradient for any mini-batch size (1 .. 2^30 - 4096 pairs): outputs identical, bit for bit, to gg_pair_grad on
 * every batch gg_pair_grad accepts, and the same in-order sums above GG_MAX_BATCH (csrc/grad_multi.cu).  Up to
 * GG_MAX_BATCH pairs without flags it runs gg_pair_grad's one-CTA kernel; otherwise a multi-CTA path that needs
 * `scratch` (device, 256-byte aligned, at least gg_pair_grad_scratch_bytes(n_pairs, ld) bytes).  uniq_ids, grad_rows
 * and grad_bias hold 2 * n_pairs entries.  gg_pair_grad_scratch_bytes is a host-only size computation. */
#define GG_GRAD_MULTI_CTA 1   /* flags: use the multi-CTA path even when n_pairs <= GG_MAX_BATCH (tests / A-B) */
int gg_pair_grad_scratch_bytes(int32_t n_pairs, int32_t ld, int64_t *bytes);
int gg_pair_grad_ex(int32_t mode, int32_t n_pairs, int32_t batch_total, const int32_t *node_id,
                    const int32_t *node_neighbor_id, const float *aux, const float *emb, const float *bias,
                    int32_t ld, float lambda, int32_t *n_unique, int32_t *uniq_ids, float *grad_rows,
                    float *grad_bias, int32_t *row_slot, void *scratch, int64_t scratch_bytes,
                    int32_t flags, void *stream);

/* Data-parallel step: merge the compact gradients of `world` ranks (each laid out as one buffer of
 * gg_grad_buf_floats(cap, ld) floats: rows[cap, ld] | bias[cap] | ids[cap] (int32 bits) | n_unique) into
 * the final unique/summed form, rank-major entry order -- every rank computes the identical result
 * from the all-gathered buffers, so replicas stay bit-identical.  Clears and re-sets row_slot. */
int64_t gg_grad_buf_floats(int32_t cap, int32_t ld);
int gg_grad_merge(int32_t world, int32_t cap, int32_t ld, const float *gathered, int32_t *n_unique,
                  int32_t *uniq_ids, float *grad_rows, float *grad_bias, int32_t *row_slot, void *stream);
/* The same merge for any number of entries (world * cap <= 2^31 - 8192; csrc/grad_multi.cu): outputs identical, bit for bit,
 * to gg_grad_merge on every input gg_grad_merge accepts.  Entry t = r * cap + s exists for s < the n_unique word of rank
 * r's block; slots are numbered in order of first occurrence over t, and every coordinate of a slot is one +0-started
 * round-to-nearest add chain over the slot's entries in rank order.  row_slot may still hold this rank's local slots on
 * entry (as gg_pair_grad[_ex] leaves them).  Up to world * cap = 16384 entries without flags it runs gg_grad_merge's
 * one-CTA kernel; otherwise a multi-CTA path (GG_GRAD_MULTI_CTA forces it) that needs `scratch` (device, 256-byte
 * aligned, at least gg_grad_merge_scratch_bytes(world, cap, ld) bytes, linear in world * cap), cap even when world > 1,
 * and `gathered` 16-byte aligned.  gg_grad_merge_scratch_bytes is a host-only size computation. */
int gg_grad_merge_scratch_bytes(int32_t world, int32_t cap, int32_t ld, int64_t *bytes);
int gg_grad_merge_ex(int32_t world, int32_t cap, int32_t ld, const float *gathered, int32_t *n_unique,
                     int32_t *uniq_ids, float *grad_rows, float *grad_bias, int32_t *row_slot, void *scratch,
                     int64_t scratch_bytes, int32_t flags, void *stream);

/* ------------------------------------------------------------------------------------------
 * Data-parallel optimizer step with its collective inside the library (csrc/comm.cu).  N replicas of the
 * per-batch loops of graph_gan.py:149-157 / 168-176: every rank computes the gradient of ITS rows of the mini-batch
 * (gg_pair_grad with batch_total), ONE ncclAllGather exchanges the compact gradients over NVLink, every rank merges
 * them in rank-major order (gg_grad_merge) and applies the same Adam sweep -- replicas stay bit-identical.
 *   gg_comm_unique_id : ncclGetUniqueId (128 bytes; rank 0 creates it, the caller broadcasts it out of band)
 *   gg_comm_init      : ncclCommInitRank on the CURRENT device -> opaque handle
 *   gg_dp_step        : the whole step on `stream` (node_id / node_neighbor_id / aux: the WHOLE batch, device, identical
 *                       on all ranks; local_buf: gg_grad_buf_floats(cap, ld) floats; gathered_buf: world times that;
 *                       cap >= 2 * ceil(n_pairs / world))
 *   gg_dp_train_steps : gg_dp_step for every start of a (host) shuffled start list, enqueued from C; beta powers as in
 *                       gg_train_steps
 * NCCL is dlopen-ed at first use (the process's already-loaded libnccl.so.2 if there is one).
 * ------------------------------------------------------------------------------------------ */
int gg_comm_unique_id(void *id128);
int gg_comm_init(const void *id128, int32_t rank, int32_t world, void **comm_out);
int gg_comm_destroy(void *comm);
int gg_comm_info(void *comm, int32_t *rank, int32_t *world, int32_t *nccl_version, uint64_t *collectives);
/* Peer-memory transport for the same step (optional; NVLink P2P through CUDA IPC, one process per GPU): every rank
 * creates an exchange buffer (gg_comm_p2p_export -> 64-byte cudaIpcMemHandle_t), the caller all-gathers the handles,
 * gg_comm_p2p_connect maps the peers' buffers.  With it, gg_dp_step runs the gradient AND the exchange in one kernel
 * (stores into every peer's buffer + a release flag) and the merge kernel waits on the flags: no collective call per step.
 * capacity_floats >= world * gg_grad_buf_floats(cap, ld).  gg_comm_use_p2p switches between the two transports. */
int gg_comm_p2p_export(void *comm, int64_t capacity_floats, void *handle64);
int gg_comm_p2p_connect(void *comm, const void *all_handles);
int gg_comm_use_p2p(void *comm, int32_t on);
int gg_dp_step(void *comm, int32_t mode, int32_t n_pairs, const int32_t *node_id, const int32_t *node_neighbor_id,
               const float *aux, int64_t n_node, int32_t ld, float *emb, float *m_emb, float *v_emb, float *bias,
               float *m_bias, float *v_bias, float lambda, float *local_buf, float *gathered_buf, int32_t cap,
               int32_t *n_unique, int32_t *uniq_ids, float *grad_rows, float *grad_bias, int32_t *row_slot,
               float lr_t, float beta1, float beta2, float eps, void *stream);
int gg_dp_train_steps(void *comm, int32_t mode, int64_t n_rows, const int64_t *start_list, int64_t n_starts,
                      int32_t batch_size, const int32_t *node_id, const int32_t *node_neighbor_id, const float *aux,
                      int64_t n_node, int32_t ld, float *emb, float *m_emb, float *v_emb, float *bias, float *m_bias,
                      float *v_bias, float lambda, float *local_buf, float *gathered_buf, int32_t cap,
                      int32_t *n_unique, int32_t *uniq_ids, float *grad_rows, float *grad_bias, int32_t *row_slot,
                      float lr, float beta1, float beta2, float eps, float *beta1_power, float *beta2_power,
                      void *stream);
/* The data-parallel step for any batch size (1 .. 2^30 - 4096 pairs).  Up to GG_MAX_BATCH pairs without flags,
 * gg_dp_step_ex / gg_dp_train_steps_ex are gg_dp_step / gg_dp_train_steps.  Otherwise every rank computes its slice
 * with gg_pair_grad_ex (batch_total = n_pairs; one CTA up to GG_MAX_BATCH pairs per slice, multi-CTA above), runs the
 * same single ncclAllGather and merges with the multi-CTA gg_grad_merge_ex.  GG_GRAD_MULTI_CTA forces the multi-CTA
 * gradient and merge at any size.  uniq_ids / grad_rows / grad_bias hold 2 * n_pairs entries; scratch: device, 256-byte
 * aligned, at least gg_dp_scratch_bytes(world, n_pairs, ld) bytes with cap = 2 * ceil(n_pairs / world) (a larger cap
 * needs gg_grad_merge_scratch_bytes(world, cap, ld)); gg_dp_scratch_bytes is host-only, the larger of the slice
 * gradient's and the merge's scratch, which run one after the other and share the buffer.  The peer-memory transport
 * stays limited to GG_MAX_BATCH pairs: with it switched on, larger batches (or flags) return an error.
 * gg_dp_train_steps_ex lays out each step's blocks with cap = 2 * ceil(rows of the step / world). */
int gg_dp_scratch_bytes(int32_t world, int32_t n_pairs, int32_t ld, int64_t *bytes);
int gg_dp_step_ex(void *comm, int32_t mode, int32_t n_pairs, const int32_t *node_id, const int32_t *node_neighbor_id,
                  const float *aux, int64_t n_node, int32_t ld, float *emb, float *m_emb, float *v_emb, float *bias,
                  float *m_bias, float *v_bias, float lambda, float *local_buf, float *gathered_buf, int32_t cap,
                  int32_t *n_unique, int32_t *uniq_ids, float *grad_rows, float *grad_bias, int32_t *row_slot,
                  float lr_t, float beta1, float beta2, float eps, void *scratch, int64_t scratch_bytes, int32_t flags,
                  void *stream);
int gg_dp_train_steps_ex(void *comm, int32_t mode, int64_t n_rows, const int64_t *start_list, int64_t n_starts,
                         int32_t batch_size, const int32_t *node_id, const int32_t *node_neighbor_id, const float *aux,
                         int64_t n_node, int32_t ld, float *emb, float *m_emb, float *v_emb, float *bias, float *m_bias,
                         float *v_bias, float lambda, float *local_buf, float *gathered_buf, int32_t cap,
                         int32_t *n_unique, int32_t *uniq_ids, float *grad_rows, float *grad_bias, int32_t *row_slot,
                         float lr, float beta1, float beta2, float eps, float *beta1_power, float *beta2_power,
                         void *scratch, int64_t scratch_bytes, int32_t flags, void *stream);

/* K3: TF1.8 AdamOptimizer sparse apply == dense decay (generator.py:30-31,
 * discriminator.py:31-32): m <- b1*m (+ (1-b1) g on touched rows), v likewise, then for ALL
 * rows var -= lr_t * m / (sqrt(v) + eps).  Resets row_slot to -1. */
/* Selects the kernel behind gg_adam_apply (identical results): "ldg" per-thread loads (default), "tma" / "tma256x2" /
 * "tma512x3" cp.async.bulk pipeline with a CTA barrier per tile, "ws16" / "ws8" warp-specialised cp.async.bulk pipeline.
 * The environment variable GG_ADAM_PATH sets the initial choice. */
int gg_set_adam_path(const char *name);
int gg_adam_apply(int64_t n_node, int32_t ld, float *emb, float *m_emb, float *v_emb, float *bias,
                  float *m_bias, float *v_bias, const int32_t *n_unique, const int32_t *uniq_ids,
                  const float *grad_rows, const float *grad_bias, int32_t *row_slot, float lr_t,
                  float beta1, float beta2, float eps, void *stream);

/* The same TF1.8 Adam step from a dense fp64 gradient (the exact game's steps, DESIGN.md section 5.5): acc_emb
 * [n_node, ld] and acc_bias [n_node] as gg_game_value_grad / gg_game_value_grad_d fill them.  Per element
 *     g = (float)(scale * acc + (double)lambda * (double)x)      fp64 mul, mul, add (no contraction), rounded once
 * with lambda = lambda_emb for the rows and lambda_bias for the biases, then the m / v / variable sequence of
 * gg_adam_apply for every row and every bias.  Pad columns (acc = x = 0) stay exactly 0.  Refuses NULL pointers,
 * n_node <= 0, an unsupported ld and a non-finite scale.  One launch. */
int gg_adam_apply_dense(int64_t n_node, int32_t ld, float *emb, float *m_emb, float *v_emb, float *bias,
                        float *m_bias, float *v_bias, const double *acc_emb, const double *acc_bias,
                        double scale, float lambda_emb, float lambda_bias, float lr_t,
                        float beta1, float beta2, float eps, void *stream);

/* The inner training loop of graph_gan.py:149-157 / 168-176: for each start in start_list (host array, already
 * shuffled by the caller): one optimizer step on rows [start, min(start + batch_size, n_rows)) of the device
 * arrays node_id / node_neighbor_id / aux -- i.e. gg_pair_grad + gg_adam_apply per step, enqueued from C so that
 * the per-step cost is two kernel launches, not a round trip through the host language.  beta1_power/beta2_power:
 * host in/out, the AdamOptimizer's beta^t accumulators (fp32, multiplied once per step like TF's _finish). */
int gg_train_steps(int32_t mode, int64_t n_rows, const int64_t *start_list, int64_t n_starts, int32_t batch_size,
                   const int32_t *node_id, const int32_t *node_neighbor_id, const float *aux, int64_t n_node, int32_t ld,
                   float *emb, float *m_emb, float *v_emb, float *bias, float *m_bias, float *v_bias, float lambda,
                   int32_t *n_unique, int32_t *uniq_ids, float *grad_rows, float *grad_bias, int32_t *row_slot, float lr,
                   float beta1, float beta2, float eps, float *beta1_power, float *beta2_power, void *stream);
/* gg_train_steps for any batch size: gg_pair_grad_ex per step, with the caller's scratch (gg_pair_grad_scratch_bytes of
 * batch_size; may be NULL when batch_size <= GG_MAX_BATCH).  uniq_ids / grad_rows / grad_bias hold 2 * batch_size entries. */
int gg_train_steps_ex(int32_t mode, int64_t n_rows, const int64_t *start_list, int64_t n_starts, int32_t batch_size,
                      const int32_t *node_id, const int32_t *node_neighbor_id, const float *aux, int64_t n_node,
                      int32_t ld, float *emb, float *m_emb, float *v_emb, float *bias, float *m_bias, float *v_bias,
                      float lambda, int32_t *n_unique, int32_t *uniq_ids, float *grad_rows, float *grad_bias,
                      int32_t *row_slot, float lr, float beta1, float beta2, float eps, float *beta1_power,
                      float *beta2_power, void *scratch, int64_t scratch_bytes, void *stream);

/* The same loop as gg_train_steps in ONE cooperative launch (persistent kernel; a ready flag and an arrival
 * counter order the gradient and the Adam sweep of every step).  start_list_dev is a DEVICE array; sync_words
 * is a device scratch of eight uint64 (zeroed by the call; [0..1] flag and counter, [2..5] diagnostic: CTA 0's
 * clock cycles in gradient / sweep / wait, and the number of steps).  Bit-identical results. */
int gg_train_loop(int32_t mode, int64_t n_rows, const int64_t *start_list_dev, int64_t n_starts, int32_t batch_size,
                  const int32_t *node_id, const int32_t *node_neighbor_id, const float *aux, int64_t n_node, int32_t ld,
                  float *emb, float *m_emb, float *v_emb, float *bias, float *m_bias, float *v_bias, float lambda,
                  int32_t *n_unique, int32_t *uniq_ids, float *grad_rows, float *grad_bias, int32_t *row_slot, float lr,
                  float beta1, float beta2, float eps, float *beta1_power, float *beta2_power, uint64_t *sync_words,
                  void *stream);

/* The same loop with ONE inter-CTA barrier per step (csrc/steps.cu: train_fused_kernel): every CTA rebuilds the
 * mini-batch's forward pass and entry lists, sweeps the rows it owns and accumulates their gradient on the fly;
 * parameters ping-pong between (emb, bias) and the caller's second buffers (emb2 [N, ld], bias2 [N]); the result is
 * always left in (emb, bias).  For graphs whose (E, m, v) stay in L2; returns an error when the per-CTA row table
 * does not fit in shared memory.  grad_rows / uniq_ids / row_slot are not used.  Bit-identical to gg_train_steps. */
int gg_train_fused(int32_t mode, int64_t n_rows, const int64_t *start_list_dev, int64_t n_starts, int32_t batch_size,
                   const int32_t *node_id, const int32_t *node_neighbor_id, const float *aux, int64_t n_node, int32_t ld,
                   float *emb, float *m_emb, float *v_emb, float *bias, float *m_bias, float *v_bias, float *emb2,
                   float *bias2, float lambda, float lr, float beta1, float beta2, float eps, float *beta1_power,
                   float *beta2_power, uint64_t *sync_words, void *stream);

/* ------------------------------------------------------------------------------------------
 * End-of-epoch dump and quality line on the device (csrc/eval.cu).  Replaces the text round trip of
 * write_embeddings_to_file (graph_gan.py:293-306) -> utils.read_embeddings (utils.py:57-67) ->
 * LinkPredictEval.eval_link_prediction (src/evaluation/link_prediction.py:19-38).
 *   gg_pair_dot_f64  : out[k] = float64 dot of rows node_id[k], node_neighbor_id[k] (np.dot on the re-read rows)
 *   gg_link_pred_acc : out2[0] = accuracy of (score >= np.median(score)) against labels [1]*(n/2) + [0]*(n - n/2),
 *                      out2[1] = the median; score / out2: device float64.  Any NaN score makes the median NaN and
 *                      the accuracy (n - n/2) / n, as np.median and the >= comparison give them
 *   gg_unpad_rows    : dense [N, n_emb] fp32 copy of the padded [N, ld] rows (payload of the binary dump)
 * ------------------------------------------------------------------------------------------ */
int gg_pair_dot_f64(int64_t n_pairs, const int32_t *node_id, const int32_t *node_neighbor_id, const float *emb,
                    int32_t ld, double *out, void *stream);
int gg_link_pred_acc(int64_t n, const double *score, double *out2, void *stream);
int gg_unpad_rows(int64_t n_node, int32_t ld, int32_t n_emb, const float *emb, float *out, void *stream);

/* get_node_pairs_from_path (graph_gan.py:272-291) for a batch of recorded paths.
 * pair_ptr: device [W+1] (out, exclusive scan of per-path pair counts). */
int gg_window_pairs(int64_t n_walks, const int32_t *paths, const int32_t *path_len, int32_t max_path,
                    int32_t window, int64_t *pair_ptr, int32_t *node_1, int32_t *node_2,
                    int64_t *n_pairs_out, int64_t capacity, void *stream);

#ifdef __cplusplus
}
#endif
#endif
