/* TEST INFRASTRUCTURE -- C inner loops of the CPU oracle (oracle/cluster_oracle.py).
 *
 * These restate, with an explicitly DEFINED floating-point order ("vk arithmetic
 * v1", DESIGN.md section 3), the tensor expressions of the reference clusterer:
 *   ok_normalize_rows  <- vamb/cluster.py:653-669  (_normalize)
 *   ok_dists           <- vamb/cluster.py:672-676  (_calc_distances)
 *   ok_sample          <- vamb/cluster.py:619-629  (sample_medoid body)
 *   ok_hist            <- vamb/cluster.py:457-481  (find_threshold head)
 * The reference evaluates them with MKL sgemv / ATen reductions whose summation
 * order is undocumented; the CUDA kernels in vamb_b200/csrc implement exactly the
 * order written here, so GPU-vs-oracle parity is bit-exact by construction and
 * oracle-vs-reference parity is checked on the golden fixtures (tests/golden).
 *
 * Build: gcc -O2 -fPIC -shared -ffp-contract=off -mfma (oracle/build.py).
 * -ffp-contract=off: no a*b+c is fused unless written as fmaf().
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

#define OK_EXPORT __attribute__((visibility("default")))

/* dot product in "8-lane" order: chunk c (elements 4c..4c+3) belongs to lane c&7,
 * each lane runs one fmaf chain over its chunks in increasing c, the eight lane
 * sums are combined by an xor-butterfly (1, 2, 4). */
static inline float dot8(const float *x, const float *q, int d) {
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    int nchunk = (d + 3) >> 2;
    for (int c = 0; c < nchunk; ++c) {
        int j = c & 7;
        int k0 = c << 2;
        int k1 = k0 + 4 < d ? k0 + 4 : d;
        float a = acc[j];
        for (int k = k0; k < k1; ++k) a = fmaf(x[k], q[k], a);
        acc[j] = a;
    }
    float s0 = acc[0] + acc[1], s1 = acc[2] + acc[3];
    float s2 = acc[4] + acc[5], s3 = acc[6] + acc[7];
    float t0 = s0 + s1, t1 = s2 + s3;
    return t0 + t1;
}

/* cluster.py:666-668.  Zero rows become 1/D; row /= (norm * sqrt(2)).
 * norm = (float)sqrt(sum_k (double)x_k^2), k ascending (products exact in double). */
OK_EXPORT void ok_normalize_rows(float *m, int64_t n, int d) {
    const float sqrt2 = (float)1.4142135623730951; /* (float)(2**0.5) */
    for (int64_t i = 0; i < n; ++i) {
        float *x = m + i * (int64_t)d;
        int allzero = 1;
        for (int k = 0; k < d; ++k)
            if (x[k] != 0.0f) { allzero = 0; break; }
        if (allzero) {
            float v = (float)(1.0 / (double)d);
            for (int k = 0; k < d; ++k) x[k] = v;
        }
        double ss = 0.0;
        for (int k = 0; k < d; ++k) ss += (double)x[k] * (double)x[k];
        float nrm = (float)sqrt(ss);
        float den = nrm * sqrt2;
        for (int k = 0; k < d; ++k) x[k] = x[k] / den;
    }
}

/* cluster.py:674-675: dists = 0.5 - M @ M[idx]; dists[idx] = 0 */
OK_EXPORT void ok_dists(const float *m, int64_t n, int d, int64_t idx, float *out) {
    const float *q = m + idx * (int64_t)d;
    for (int64_t i = 0; i < n; ++i) out[i] = 0.5f - dot8(m + i * (int64_t)d, q, d);
    out[idx] = 0.0f;
}

/* cluster.py:625-629.  within = dists <= radius (fp32 compare); indices ascending;
 * density = sum len_i * (radius - d_i).  closeness is a multiple of 2^-29 (radius is
 * 0.05f), lengths are integers, so the sum is accumulated EXACTLY in integers, in units of
 * 2^-29 (order independent): density = hi * 4096 + lo with lo = sum len * (c & 4095),
 * hi = sum len * (c >> 12).  Returns the count. */
OK_EXPORT int64_t ok_sample(const float *dists, const float *lens, int64_t n, float radius,
                            int64_t *idx_out, uint64_t *density_lo_hi) {
    int64_t cnt = 0;
    uint64_t lo = 0, hi = 0;
    for (int64_t i = 0; i < n; ++i) {
        float dd = dists[i];
        if (dd <= radius) {
            float c = radius - dd;
            uint64_t cq = (uint64_t)((double)c * 536870912.0); /* exact: c is k * 2^-29 */
            lo += (uint64_t)lens[i] * (cq & 4095u);
            hi += (uint64_t)lens[i] * (cq >> 12);
            if (idx_out) idx_out[cnt] = i;
            ++cnt;
        }
    }
    density_lo_hi[0] = lo;
    density_lo_hi[1] = hi;
    return cnt;
}

/* cluster.py:457 and :467-481.  n_lt = #(d < 0.05f).  Histogram of d in [0, 0.3f]
 * (d <= 0.3f picked at :467, torch.histogram drops d < 0), bin = upper_bound over the
 * 61 fp32 edges - 1, last bin right-inclusive; weights = lengths summed exactly. */
OK_EXPORT int64_t ok_hist(const float *dists, const float *lens, int64_t n, const float *edges,
                          int nbins, float medoid_radius, uint64_t *hist) {
    int64_t n_lt = 0;
    memset(hist, 0, sizeof(uint64_t) * (size_t)nbins);
    float lo = edges[0], hi = edges[nbins];
    for (int64_t i = 0; i < n; ++i) {
        float dd = dists[i];
        if (dd < medoid_radius) ++n_lt;
        if (!(dd <= hi) || dd < lo) continue;
        int a = 0, b = nbins + 1; /* upper_bound over edges[0..nbins] */
        while (a < b) {
            int mid = (a + b) >> 1;
            if (edges[mid] <= dd) a = mid + 1; else b = mid;
        }
        int pos = a - 1;
        if (pos == nbins) pos = nbins - 1;
        hist[pos] += (uint64_t)lens[i];
    }
    return n_lt;
}

/* members = indices with d <= thr, ascending (cluster.py:640-650) */
OK_EXPORT int64_t ok_smaller(const float *dists, int64_t n, float thr, int64_t *idx_out) {
    int64_t cnt = 0;
    for (int64_t i = 0; i < n; ++i)
        if (dists[i] <= thr) idx_out[cnt++] = i;
    return cnt;
}

/* vambtools.py:307-321 / vambcore.overwrite_matrix: stable in-place row compaction */
OK_EXPORT int64_t ok_pack_rows(float *m, float *lens, int64_t *indices, const uint8_t *keep,
                               int64_t n, int d) {
    int64_t w = 0;
    for (int64_t i = 0; i < n; ++i) {
        if (!keep[i]) continue;
        if (w != i) {
            memmove(m + w * (int64_t)d, m + i * (int64_t)d, sizeof(float) * (size_t)d);
            lens[w] = lens[i];
            indices[w] = indices[i];
        }
        ++w;
    }
    return w;
}
