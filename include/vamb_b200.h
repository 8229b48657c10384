/* vamb_b200 -- C ABI of the H100 (sm_90a) kernels behind the vamb hot path.
 *
 * Drop-in boundary (SURVEY.md section 8b).  The reference (RasmussenLab/vamb) is
 * pure Python + PyTorch and has no FFI of its own; the functions below are what a
 * ctypes binding inside vamb/encode.py and vamb/cluster.py would bind to replace the
 * tensor expressions cited next to each entry point.  INTEGRATION.md shows the stub.
 *
 * Conventions
 *   - plain C: pointers + sizes, no torch / C++ types.  Pointers are DEVICE pointers
 *     unless the name ends in `_host` (then: pinned host memory).
 *   - every call is asynchronous on `stream` (a cudaStream_t passed as void*), except
 *     the `*_sync` entry points, which end with one cudaStreamSynchronize.
 *   - return value: 0 = ok, non-zero = failure; vk_last_error() (thread-local) has the
 *     message.  Nothing throws, nothing allocates persistent device memory: all
 *     buffers are owned by the caller (the Python host code holds them as tensors).
 *   - "vk arithmetic v1" (DESIGN.md section 3) fixes the floating-point evaluation
 *     order of every reduction so that results are bit-identical to oracle/.
 */
#ifndef VAMB_B200_H
#define VAMB_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VK_ABI_VERSION 2
#define VK_NBINS 60          /* ceil(0.3 / 0.005), vamb/cluster.py:231 */
#define VK_MAX_CAND 32       /* candidates evaluated per vk_eval_candidates launch */
#define VK_LIST_CAND 64      /* candidates evaluated per vk_eval_candidates_lists launch */
#define VK_EVAL_SUBS 4       /* copies of its device accumulators / id lists (spread by block: L2 atomic contention) */
#define VK_EVAL_SCRATCH_U64 (VK_EVAL_SUBS * VK_LIST_CAND * 16) /* uint64 words of its device accumulator scratch */
#define VK_PROBE_INLINE 2040 /* `within` ids returned inline with the probe header */

const char *vk_last_error(void);
int vk_abi_version(void);
/* sm_90a-only build: returns 0 when the current device can run these kernels. */
int vk_check_device(void);

/* ------------------------------------------------------------------ clustering */

/* Result header of one probe; lives in device memory, copied to pinned host memory.
 * All sums are exact integers, hence independent of the order of accumulation. */
typedef struct vk_probe_header {
    /* local density = sum len_i * (0.05f - d_i) over kept rows with d_i <= 0.05f, exact, in units of
     * 2^-29: c_i = (0.05f - d_i) * 2^29 is an integer < 2^25; density = density_hi * 4096 + density_lo
     * with density_lo = sum len_i * (c_i & 4095), density_hi = sum len_i * (c_i >> 12).  Exact while the
     * total sequence length is below 2^50. */
    uint64_t density_lo;
    uint64_t density_hi;
    uint64_t hist[VK_NBINS];  /* sum of len_i per distance bin over kept rows with 0 <= d_i <= 0.3f       */
    int32_t n_within;         /* kept rows with d <= 0.05f  (cluster.py:625)                               */
    int32_t n_lt;             /* kept rows with d <  0.05f  (cluster.py:457, loner test)                   */
    int32_t n_nl;             /* kept rows with d <= nl_radius (entries appended to the neighbour list)    */
    int32_t rank;             /* kept rows with row index < medoid row (the reference's packed index)      */
    int32_t within[VK_PROBE_INLINE]; /* unordered row ids with d <= 0.05f (first VK_PROBE_INLINE of them)  */
} vk_probe_header;

/* vamb/cluster.py:653-669 (_normalize), in place: zero rows -> 1/D, row /= (|row| * sqrt 2). */
int vk_normalize_rows(float *matrix, int64_t n, int d, void *stream);

/* Per-row check that 2*|row|^2 is within `tol` of 1; *n_bad (device int32) receives the count. */
int vk_check_normalized(const float *matrix, int64_t n, int d, float tol, int32_t *n_bad, void *stream);

/* One seed->all-contigs pass: vamb/cluster.py:672-676 (_calc_distances) fused with
 * :619-629 (within-radius set + local density), :457-481 (loner count + weighted
 * histogram) and the collection of the neighbour list {kept rows with d <= nl_radius}
 * that vk_eval_candidates / vk_select_members consume.  `edges` = the 61 fp32 bin edges.
 * `hdr` is zeroed by the call.  within ids beyond VK_PROBE_INLINE go to `within_overflow`
 * (capacity n) at positions [VK_PROBE_INLINE, n_within). */
int vk_probe(const float *matrix, const float *lengths, const uint8_t *kept, int64_t n, int d,
             int64_t medoid_row, float nl_radius, const float *edges,
             vk_probe_header *hdr, int32_t *within_overflow,
             int32_t *nl_rows, float *nl_dists, void *stream);

/* vk_probe + copy of the header to `hdr_host` (pinned) + stream synchronize. */
int vk_probe_sync(const float *matrix, const float *lengths, const uint8_t *kept, int64_t n, int d,
                  int64_t medoid_row, float nl_radius, const float *edges,
                  vk_probe_header *hdr, int32_t *within_overflow,
                  int32_t *nl_rows, float *nl_dists, vk_probe_header *hdr_host, void *stream);

/* Same pass with a "mapped" completion: the last block copies the header into PINNED host memory
 * (`hdr_pinned`, device-visible), leaves the device accumulators of `hdr` zeroed for the next call and sets
 * `*done_flag_pinned = seq`; the call returns once the host has seen the flag.  `hdr` must be all zero before
 * the first call, `*done_ticket` (device) zero.  One launch per probe instead of memset + kernel + copy +
 * stream synchronisation.  `work_counter` (device int32, zero before the first call, left zero; NULL = static
 * striding): the blocks draw their 256-row work units from it, so faster SMs scan more of the matrix.
 * Used by the native cluster driver (vk_cluster_next). */
int vk_probe_mapped(const float *matrix, const float *lengths, const uint8_t *kept, int64_t n, int d,
                    int64_t medoid_row, float nl_radius, const float *edges, vk_probe_header *hdr,
                    int32_t *within_overflow, int32_t *nl_rows, float *nl_dists, vk_probe_header *hdr_pinned,
                    int32_t *done_ticket, int32_t *done_flag_pinned, int32_t seq, int32_t *work_counter, void *stream);

/* Local densities of up to VK_MAX_CAND candidate medoids in one pass over the neighbour
 * list (the <= maxsteps sample_medoid calls of one wander_medoid round,
 * vamb/cluster.py:427-448, whose densities are independent of each other).  Only list
 * entries with nl_dists <= prune_radius are visited (see DESIGN.md: a row within 0.05 of
 * a candidate that is itself within 0.05 of the medoid lies within 0.19 of the medoid).
 * out_host (pinned host, 3*VK_MAX_CAND uint64) = density_lo[k], then density_hi[k], then counts[k].  Ends with a stream synchronize. */
int vk_eval_candidates_sync(const float *matrix, const float *lengths, int d,
                            const int32_t *nl_rows, const float *nl_dists, int32_t n_nl,
                            float prune_radius, const int32_t *cand_rows_host, int n_cand,
                            uint64_t *out_dev, uint64_t *out_host, void *stream);

/* vk_eval_candidates_sync through the mapped completion (out_dev all zero on entry, left zeroed). */
int vk_eval_candidates_mapped(const float *matrix, const float *lengths, int d, const int32_t *nl_rows,
                              const float *nl_dists, int32_t n_nl, float prune_radius, const int32_t *cand_rows_host,
                              int n_cand, uint64_t *out_dev, uint64_t *out_pinned, int32_t *done_ticket,
                              int32_t *done_flag_pinned, int32_t seq, void *stream);

/* Candidate evaluation that also returns what is needed to MOVE the medoid to a winning candidate without another
 * full scan (native driver): the ids of the rows within 0.05 of candidate k (its `cluster`, vamb/cluster.py:626) are
 * written to within_pinned[k * within_cap ...] (pinned host memory; entries beyond within_cap are dropped, the count
 * still tells), and out_pinned (4 * VK_LIST_CAND uint64) = density_lo[k] | density_hi[k] | counts[k] | fp32 bits of
 * d(candidate k, base_row).  `base_row` = the medoid whose neighbour list (radius nl_radius = 0.3) is passed in: the list
 * covers the whole 0.05-neighbourhood of a candidate iff d(candidate, base) <= 0.12 (angles add: acos(0.76) +
 * acos(0.9) = acos(0.4)), which the caller checks.  The id list of candidate k is only published if its density exceeds
 * min_density = min_density_hi * 4096 + min_density_lo (the current medoid's: nothing else can be moved to; 0, 0 = all).  Mapped completion as vk_eval_candidates_mapped (out_dev:
 * VK_EVAL_SCRATCH_U64 uint64 of device scratch, all zero on entry, left zeroed; n_cand <= VK_LIST_CAND). */
int vk_eval_candidates_lists(const float *matrix, const float *lengths, int d, const int32_t *nl_rows,
                             const float *nl_dists, int32_t n_nl, float prune_radius, const int32_t *cand_rows_host,
                             int n_cand, int32_t base_row, uint64_t min_density_hi, uint64_t min_density_lo,
                             uint64_t *out_dev, uint64_t *out_pinned,
                             int32_t *within_dev /* device scratch [VK_EVAL_SUBS * VK_LIST_CAND * within_cap] */, int32_t *within_pinned,
                             int32_t within_cap, int32_t *done_ticket, int32_t *done_flag_pinned, int32_t seq, void *stream);

/* vamb/cluster.py:640-650 (_smaller_indices) + :308-309 (kept_mask[point] = 0):
 * appends orig_ids[row] of every neighbour-list entry with d <= threshold to `members`
 * (unordered), clears kept[row], returns the count through members_host[0] and the ids
 * through members_host[1..] (pinned, capacity_host int32 entries; ids beyond that stay in
 * `members` on the device).  Ends with a stream synchronize. */
int vk_select_members_sync(const int32_t *nl_rows, const float *nl_dists, int32_t n_nl, float threshold,
                           const int32_t *orig_ids, uint8_t *kept, int32_t *members /* [1 + n_nl] */,
                           int32_t *members_host, int32_t capacity_host, void *stream);

/* kept[rows[i]] = 0 for i < n (rows: device int32). */
int vk_mask_clear(uint8_t *kept, const int32_t *rows, int32_t n, void *stream);

/* vamb/cluster.py:318-335 (pack) / vambcore.overwrite_matrix: stable row compaction of
 * (matrix, lengths, orig_ids) by `kept` into the *_out buffers; kept_out[0..n_out) = 1.
 * tile_scratch: int32[2 + ceil(n / 1024)].  *n_out_host (pinned int64) receives the new
 * row count.  Ends with a stream synchronize. */
int vk_compact_rows_sync(const float *matrix, const float *lengths, const int32_t *orig_ids,
                         const uint8_t *kept, int64_t n, int d,
                         float *matrix_out, float *lengths_out, int32_t *orig_out, uint8_t *kept_out,
                         int32_t *tile_scratch, int64_t *n_out_host, void *stream);

/* Full distance vector (vamb/cluster.py:672-676) -- used by tests and the roofline bench. */
int vk_distances(const float *matrix, int64_t n, int d, int64_t medoid_row, float *dists, void *stream);


/* The step before the path (SURVEY 8f-4): vamb/parsecontigs.py:141-150 Composition._project -- per contig the 256
 * four-mer counts become frequencies (row / rowsum; all-zero rows stay zero), shifted by -1/256 and multiplied by the
 * 256 x n_out projection kernel (n_out = 103; the caller passes the reference's kernel matrix, row-major [256][n_out]).
 * counts: device [n, 256] fp32 (not modified, unlike the reference's in-place version); out: device [n, n_out]. */
int vk_tnf_project(const float *counts, const float *kernel, float *out, int64_t n, int n_out, void *stream);

/* ------------------------------------------------------------------ native clusterer driver
 * The decision logic of vamb/cluster.py (ClusterGenerator.__next__ :298-316 and everything it
 * calls) in C++ on top of the kernels above: one foreign call per emitted cluster.  All device and
 * pinned buffers are owned by the caller; sizes as in vamb_b200/cluster.py. */
typedef struct vk_cluster_config {
    int64_t n;                 /* observations                                                          */
    int32_t d;                 /* latent width                                                          */
    int32_t maxsteps, windowsize, minsuccesses;
    float nl_radius, prune_radius;
    double pack_fraction;      /* compact the device arrays when live rows < pack_fraction * physical   */
    /* double-buffered device state (set 2 is the compaction target) */
    float *matrix, *matrix2;   /* [n, d] normalised rows                                                */
    float *lengths, *lengths2; /* [n]                                                                   */
    uint8_t *kept, *kept2;     /* [n]                                                                   */
    int32_t *orig, *orig2;     /* [n] original ids                                                      */
    int32_t *nl_rows;          /* [n]                                                                   */
    float *nl_dists;           /* [n]                                                                   */
    vk_probe_header *hdr;      /* device                                                                */
    int32_t *within_overflow;  /* [n]                                                                   */
    const float *edges;        /* [61] device                                                           */
    uint64_t *cand_out;        /* [3 * VK_MAX_CAND] device                                              */
    int32_t *members;          /* [n + 1] device                                                        */
    int32_t *tile_scratch;     /* [2 + ceil(n / 1024)] device                                           */
    vk_probe_header *hdr_host; /* pinned                                                                */
    uint64_t *cand_out_host;   /* pinned [3 * VK_MAX_CAND]                                              */
    int32_t *members_host;     /* pinned [members_host_cap]                                             */
    int32_t members_host_cap;
    int32_t seed_key_len;      /* 32-bit words of |rng_seed| (CPython random.seed(int)), >= 1           */
    const uint32_t *seed_key;  /* host                                                                  */
    const int64_t *order_host; /* host [n]: np.argsort(lengths)[::-1] (vamb/cluster.py:275)             */
    const float *normalpdf_host; /* host [31]: the smoothing kernel (vamb/cluster.py:39-73)             */
    void *stream;
} vk_cluster_config;

typedef struct vk_cluster_result {
    int64_t medoid, seed, n_members, n_remaining;
    const int64_t *members_host; /* ascending original ids; valid until the next call                  */
    double maximal_pvr, observed_pvr, radius, peak_valley_ratio; /* NaN = None                         */
    int32_t kind;                /* 0 loner, 1 fallback, 2 normal                                      */
    int32_t successes, attempts;
} vk_cluster_result;

/* A block of consecutive clusters in caller-provided HOST arrays (struct-of-arrays; `members` holds the ascending
 * original ids of cluster 0, then cluster 1, ... -- capacity n is always enough).  Fields as in vk_cluster_result. */
typedef struct vk_cluster_block {
    int64_t max_clusters;        /* in: capacity of the per-cluster arrays                                */
    int64_t n_clusters;          /* out                                                                   */
    int64_t n_members_total;     /* out: entries used in `members`                                        */
    int64_t n_remaining;         /* out: unclustered observations after the block                         */
    int64_t *medoid, *seed, *n_members; /* [max_clusters]                                                 */
    int64_t *members;            /* [n]                                                                   */
    double *maximal_pvr, *observed_pvr, *radius; /* [max_clusters], NaN = None                            */
    int32_t *kind, *successes, *attempts;        /* [max_clusters]                                        */
    double peak_valley_ratio;    /* out: the generator's pvr after the block                              */
} vk_cluster_block;

int vk_cluster_create(void **handle, const vk_cluster_config *cfg);
/* Up to blk->max_clusters calls of vk_cluster_next in ONE foreign call (vamb/__main__.py:1289-1377 consumes the
 * clusters as a stream; per-cluster Python becomes per-block NumPy).  0 = ok (n_clusters may be 0: exhausted), 1 = error. */
int vk_cluster_next_block(void *handle, vk_cluster_block *blk);
int vk_cluster_next(void *handle, vk_cluster_result *out); /* 0 = cluster, 2 = exhausted, 1 = error */
int vk_cluster_stats(void *handle, int64_t *out8);         /* probes, evals, packs, physical rows, live buffer set (0/1),
                                                              successes, attempts in the window, order_index */
int vk_cluster_timing(void *handle, double *out8);         /* host seconds in probes, evaluations, selections, packs, total;
                                                              medoid moves without a scan, re-basing probes, sum of neighbour-list sizes over evaluations */
void vk_cluster_destroy(void *handle);
int64_t vk_cluster_sizeof(int which);                      /* 0: vk_cluster_config, 1: vk_cluster_result, 2: vk_cluster_block */
/* CPython-compatible random.Random(seed).sample(range(n_i), min(n_i, k)) for each i: writes k slots per
 * call into out (unused slots = -1).  Host only; used by the CPU test-suite. */
int vk_cluster_rng_selftest(const uint32_t *key, int key_len, const int32_t *ns, int n_calls, int k, int32_t *out);

/* ------------------------------------------------------------------ VAE (vamb/encode.py) */

#define VK_VAE_MAX_LAYERS 10 /* linear layers: len(nhiddens) encoder + mu + len(nhiddens) decoder + output */
#define VK_VAE_ROW_TILE 64   /* batch rows per partial-statistics tile */

enum { VK_LAYER_HIDDEN = 0, VK_LAYER_MU = 1, VK_LAYER_OUT = 2 };   /* vk_vae_layer.kind    */
enum { VK_IN_DATA = 0, VK_IN_BN = 1, VK_IN_Z = 2 };                /* vk_vae_layer.in_kind */

/* Device-resident control block: everything a replayed CUDA graph must read at run time. */
typedef struct vk_vae_ctl {
    double d;              /* D-Adaptation distance estimate (dadaptation DAdaptAdam: group['d'])            */
    double num_w;          /* group['numerator_weighted']                                                     */
    double loss_sums[5];   /* running sums of (loss, ab, ce, sse, kld) over the steps since the last reset    */
    double wbar;           /* mean of the batch weights (the reference's [B]x[B,1] broadcast, encode.py:349)  */
    int64_t step;          /* optimiser steps taken (Philox counter)                                          */
    int64_t epoch_step0;   /* value of `step` at the start of the current epoch                               */
    int64_t n_loss_steps;  /* number of steps accumulated in loss_sums                                        */
    uint64_t seed;         /* Philox key / Feistel key base                                                   */
    int32_t epoch;         /* current epoch (selects the row permutation)                                     */
    int32_t tickets[2 * VK_VAE_MAX_LAYERS + 4]; /* last-block-done counters (self-resetting)                  */
    int32_t barrier_gen[2 * VK_VAE_MAX_LAYERS]; /* generation words of the in-kernel grid barriers (fused staging) */
} vk_vae_ctl;

/* One Linear (+ LeakyReLU + Dropout + BatchNorm1d) block, encode.py:259-295.  All pointers device. */
typedef struct vk_vae_layer {
    int32_t k_in, n_out;
    int32_t kind, in_kind;
    int64_t w_off, b_off;       /* float offsets into the parameter / gradient / optimiser arenas: W[n_out,k_in], b */
    int64_t g_off, beta_off;    /* BatchNorm weight / bias offsets (-1 when kind != hidden)                        */
    float *running_mean, *running_var;
    int64_t *num_batches_tracked;
    float *act;                 /* hidden: P = dropout(leakyrelu(x W^T + b)) [bmax, n_out]; mu: MU; out: R          */
    float *dact;                /* hidden: dL/dBN(P); mu: dL/dmu; out: dL/dR                     [bmax, n_out]      */
    double *fwd_part;           /* [ceil(bmax/ROW_TILE)][2][n_out] column sums of P and P^2 per row tile            */
    double *bwd_part;           /* [ceil(bmax/ROW_TILE)][2][n_out] column sums of dH and dH*Phat per row tile        */
    float *bn_a, *bn_c;         /* BN(P) = P * bn_a + bn_c  (batch statistics in training, running in eval)         */
    float *bn_mean, *bn_rstd;   /* batch mean and 1/sqrt(var + eps) of the current step                             */
    float *bn_m1, *bn_m2;       /* mean_b dH and mean_b dH*Phat of the current step                                 */
    float *bn_bA, *bn_bB, *bn_bC; /* dL/dY = sgn * (bA*dH + bB*P + bC): folded BatchNorm/dropout backward constants  */
    /* Tensor-core operand staging: plain K-major arrays, zero padded (rows to 128, K to 32); `hi` is
     * the fp32 value (the tensor core reads its top 19 bits), `lo` the tf32 remainder. */
    float *xop_hi, *xop_lo;     /* layer input            [bmax, ld = round32(k_in)]       A of the forward GEMM    */
    float *xt_hi, *xt_lo;       /* its transpose + a row of ones [round128(k_in + 1), bmax] B of wgrad              */
    float *dy_hi, *dy_lo;       /* dL/dY                  [bmax, ld = round32(n_out)]      A of dgrad               */
    float *dyt_hi, *dyt_lo;     /* its transpose          [round128(n_out), bmax]          A of wgrad               */
    float *w_hi, *w_lo;         /* W                      [round128(n_out), round32(k_in)] B of the forward GEMM    */
    float *wt_hi, *wt_lo;       /* W^T                    [round128(k_in), round32(n_out)] B of dgrad               */
} vk_vae_layer;

typedef struct vk_vae {
    int32_t n_layers, nsamples, ntnf, nlatent, d_in, bmax;
    float dropout, slope;
    float ce_w, ab_w, sse_w, kld_w;     /* encode.py:334-343 */
    int64_t n_rows;                     /* rows of the resident dataset                       */
    const float *data;                  /* [n_rows, d_in] = depths | tnf | total abundance    */
    const float *weights;               /* [n_rows] contig weights (encode.py:122-126)        */
    int64_t n_params;
    float *params, *grads, *exp_avg, *exp_avg_sq, *s; /* flat arenas, module.parameters() order */
    float *z;                           /* [bmax, nlatent] mu + eps                            */
    int64_t *batch_rows;                /* [bmax] dataset row of every batch row               */
    double *opt_part;                   /* [2 * ceil(n_params / 1024) + bmax / 32 + 8] optimiser block partials, then the batch-weight partials */
    double *loss_part;                  /* [4 * ceil(bmax / 32) * 4 + 64] loss block partials (4 per 8 rows) */
    vk_vae_ctl *ctl;
    vk_vae_layer layers[VK_VAE_MAX_LAYERS];
    int32_t data_ld;                    /* floats per dataset row (>= d_in; a multiple of 4 keeps rows 16-byte aligned) */
    int32_t tc_min_batch;               /* batches >= this run the GEMMs on wgmma (3xTF32); 0 = never              */
    int64_t grad_slab;                  /* floats between the split-K gradient slabs of `grads`                    */
    int32_t n_grad_slabs;               /* slabs allocated in `grads` (>= 1)                                       */
    int32_t staging;                    /* tensor-core operand staging: 0 = fused into the producing kernels' epilogues
                                           (grid barrier; falls back when a grid exceeds the SM count), 1 = prep kernels */
    int32_t use_tma;                    /* 1 = the weight operand (B) of the forward / dgrad GEMMs is fetched by TMA
                                           (cp.async.bulk.tensor, 128B swizzle; needs w_lo / wt_lo), 0 = cp.async ring  */
    int32_t wgrad_flush;                /* 1 = wgrad sums every 128 batch rows into fp32 registers (two alternating tensor-memory
                                           accumulators) instead of one truncating accumulation chain per 512-row split;
                                           2 = also the forward GEMMs in training (evaluation always uses the flushed form) */
} vk_vae;

/* Optional host-injected randomness for parity tests (all device pointers, NULL = on-device RNG). */
typedef struct vk_vae_inject {
    const int64_t *batch_idx;                   /* [batch] dataset rows; NULL = epoch permutation       */
    const float *eps;                           /* [batch, nlatent] reparameterisation noise             */
    const uint8_t *keep[VK_VAE_MAX_LAYERS];     /* [batch, n_out] dropout keep-masks per hidden layer    */
} vk_vae_inject;

int64_t vk_vae_sizeof(int which); /* 0: vk_vae, 1: vk_vae_layer, 2: vk_vae_ctl, 3: vk_vae_inject */

/* One optimiser step (encode.py:401-419): batch gather, forward (:259-314), loss (:316-357) and
 * its backward, D-Adaptation Adam update (dadaptation.DAdaptAdam.step).  `net` and `inject` are HOST
 * structs holding device pointers.  Stream-ordered, graph-capturable, no host synchronisation. */
int vk_vae_train_step(const vk_vae *net, int batch, const vk_vae_inject *inject, void *stream);

/* Forward only on rows [row0, row0 + batch) of the resident dataset (or inject->batch_idx).
 * training != 0: batch statistics + dropout (encode.py:306-314 in train mode) and the loss kernel;
 * training == 0: running statistics, no dropout.  Results stay in layer.act buffers. */
int vk_vae_forward(const vk_vae *net, int64_t row0, int batch, int training, int with_loss,
                   const vk_vae_inject *inject, void *stream);

/* encode.py:442-484: eval-mode mu of rows [row0, row0 + n) with the low `mask_bits` mantissa bits
 * cleared (vambtools.py:324-330), written to latent_out[n, nlatent] (device). */
int vk_vae_encode(const vk_vae *net, int64_t row0, int64_t n, int mask_bits, float *latent_out, void *stream);

/* Once per process and device, outside any stream capture: creates the side stream / events on which a
 * training step runs its off-critical-path work (weight staging, loss bookkeeping).  Optional: without it
 * everything runs on the caller's stream. */
int vk_vae_init_device(void);

/* Eval-mode BatchNorm affine from the running statistics into bn_a / bn_c. */
int vk_vae_prepare_eval(const vk_vae *net, void *stream);

/* Standalone D-Adaptation Adam step on the arenas (used after a gradient all-reduce). */
int vk_vae_dadapt_step(const vk_vae *net, void *stream);

/* vk_vae_train_step with a CUDA event before every launch: ms_out_host[i] = device time of launch i,
 * kinds_out_host[i] = 0 batch rows | 1 forward layer | 2 loss | 3 backward layer | 4 optimiser |
 * 5 operand staging.  Synchronises. */
int vk_vae_profile_step(const vk_vae *net, int batch, const vk_vae_inject *inject, float *ms_out_host,
                        int *kinds_out_host, int capacity, int *n_launches, void *stream);

/* Backward + gradients only (no optimiser): used by the multi-GPU path and by the tests. */
int vk_vae_grad_step(const vk_vae *net, int batch, const vk_vae_inject *inject, void *stream);

/* Stand-alone check of the PRODUCTION wgmma 3xTF32 main loop (tc::ws_mainloop -- the loop of the layer kernels):
 * C[M,N] = A * B^T over k-tiles [kt0, kt0 + nk) of 32.  A_lane: the 128-row operand in the lane-major staging layout
 * (vk_lane_major_index), zero padded to whole 128-row panels; B: plain row-major [rows][ldb], zero padded to whole
 * tile_n-row tiles; lda, ldb multiples of 32; tile_n (output columns per CTA) a multiple of 16 in [16, 128].
 * B_lo != NULL selects the TMA-fed B operand (cp.async.bulk.tensor through 128B-swizzled tensor maps), B_lo holding the
 * tf32 remainders x - trunc13(x) of B -- the way the forward / dgrad GEMMs fetch the weights staged by prep_weights.
 * flush != 0 (B_lo == NULL) selects the wgrad variant: the accumulation chain is cut every 4 k-tiles (128 rows). */
int vk_tc_gemm_test(const float *A_lane, int lda, const float *B, const float *B_lo, int ldb, float *C, int M, int N,
                    int tile_n, int kt0, int nk, int flush, void *stream);

/* Host-side: float offset of element (r, k) of an A-role operand in the "lane-major" staging layout
 * (128-row panels; each 32-wide k-tile of a panel is one 16 KB block [k/4][row][k%4]); ld = floats per row,
 * a multiple of 32.  Same footprint as the row-major [rows][ld] array.  (Layout contract of the tensor-core
 * path, checked by the CPU tests.) */
int64_t vk_lane_major_index(int r, int k, int ld);

#ifdef __cplusplus
}
#endif
#endif /* VAMB_B200_H */
