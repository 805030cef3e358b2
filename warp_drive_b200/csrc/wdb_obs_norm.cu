// wdb_obs_norm.cu -- running observation statistics and the normalization they drive
// (include/wdb200.h, wdb_obs_*).
//
// A moments update is two launches and no host wait.  The partial pass splits the batch's rows
// into fixed ranges, one CTA each, and writes one record (n, mean[F], M2[F]) per range: every
// thread runs float64 Welford over its own rows, then the CTA merges its threads' moments in a
// fixed tree (Chan et al.).  The merge pass folds the records in record order into the running
// (count, mean, M2) and rewrites the float32 shift and scale the forwards read.  No float
// atomics and no order that depends on scheduling, so the statistics are bit-reproducible run
// to run.  A record is [n, mean_0 .. mean_{F-1}, M2_0 .. M2_{F-1}] in float64; the same layout
// carries a rank's batch moments between GPUs.
#include <cmath>

#include "wdb_common.cuh"
#include "wdb_obs_norm.cuh"

using namespace wdb;

namespace {

constexpr int kThreads = 256;
constexpr long long kMaxRecords = 512;      // per-CTA records of one batch
constexpr long long kRowsPerRecord = 1024;  // at least, before the cap above
constexpr int kMaxFeatures = 1 << 16;

__host__ __device__ inline long long n_records(long long rows) {
  const long long p = (rows + kRowsPerRecord - 1) / kRowsPerRecord;
  return p < 1 ? 1 : (p > kMaxRecords ? kMaxRecords : p);
}

// (na, ma, m2a) <- (na, ma, m2a) merged with (nb, mb, m2b) (Chan et al.); an empty side
// leaves the other exactly as it is
__device__ __forceinline__ void chan(double &na, double &ma, double &m2a, double nb, double mb,
                                     double m2b) {
  if (nb == 0.0) return;
  if (na == 0.0) {
    na = nb; ma = mb; m2a = m2b;
    return;
  }
  const double n = na + nb, d = mb - ma;
  ma = ma + d * (nb / n);
  m2a = m2a + m2b + d * d * (na * nb / n);
  na = n;
}

// one Welford step of the k-th value v (k counted here)
__device__ __forceinline__ void welford(double v, long long &k, double &mean, double &m2) {
  k++;
  const double inv = 1.0 / (double)k;          // off the chain through mean
  const double d = v - mean;
  mean = fma(d, inv, mean);
  m2 = fma(d, v - mean, m2);
}

// grid (records, feature tiles).  A tile is FT = min(F, 256) features; the CTA's threads are
// L = 256 / FT row lanes of FT features (thread t: feature t % FT, lane t / FT), so a warp reads
// consecutive words of the row-major batch.  Lane l takes rows begin + l, begin + l + L, ...
__global__ void __launch_bounds__(kThreads)
obs_moments_partial_kernel(const float *__restrict__ x, long long rows, int F,
                           double *__restrict__ records) {
  __shared__ double s_n[kThreads], s_mean[kThreads], s_m2[kThreads];
  const long long P = gridDim.x, rec = blockIdx.x;
  const long long begin = rec * rows / P, end = (rec + 1) * rows / P;
  const int FT = F < kThreads ? F : kThreads, L = kThreads / FT;
  const int fl = threadIdx.x % FT, lane = threadIdx.x / FT;
  const int f = blockIdx.y * FT + fl;
  const bool on = lane < L && f < F;
  double n = 0.0, mean = 0.0, m2 = 0.0;
  if (on) {
    long long k = 0, r = begin + lane;
    // eight rows' loads in flight ahead of their (serial) updates
    for (; r + 7LL * L < end; r += 8LL * L) {
      float v[8];
#pragma unroll
      for (int j = 0; j < 8; j++) v[j] = x[(r + (long long)j * L) * F + f];
#pragma unroll
      for (int j = 0; j < 8; j++) welford((double)v[j], k, mean, m2);
    }
    for (; r < end; r += L) welford((double)x[r * F + f], k, mean, m2);
    n = (double)k;
  }
  s_n[threadIdx.x] = n;
  s_mean[threadIdx.x] = mean;
  s_m2[threadIdx.x] = m2;
  __syncthreads();
  // lane l absorbs lane l + s for s = 1, 2, 4, ...: a fixed tree over the row lanes
  for (int s = 1; s < L; s *= 2) {
    if (on && lane % (2 * s) == 0 && lane + s < L) {
      const int o = threadIdx.x + s * FT;
      chan(n, mean, m2, s_n[o], s_mean[o], s_m2[o]);
      s_n[threadIdx.x] = n;
      s_mean[threadIdx.x] = mean;
      s_m2[threadIdx.x] = m2;
    }
    __syncthreads();
  }
  if (on && lane == 0) {
    double *out = records + rec * (2LL * F + 1);
    if (f == 0) out[0] = (double)(end - begin);
    out[1 + f] = mean;
    out[1 + F + f] = m2;
  }
}

// One CTA: folds records 0 .. K-1 in order into (out_record) or into the running (count, mean,
// M2), then rewrites shift and scale.  The Chan weights of record p depend only on the counts,
// so they are computed once per record (thread 0 accumulates the counts in order) and every
// feature's chain is adds and fmas, with no branch: an empty record has weights (0, 0) and
// leaves the state as it is; the first non-empty one (1, 0), which on the empty state (mean and
// M2 zero) gives the record itself.
__global__ void __launch_bounds__(kThreads)
obs_moments_merge_kernel(const double *__restrict__ records, int K, int F, double *out_record,
                         double *count, double *mean, double *m2, float *shift, float *scale) {
  extern __shared__ double s_w[];               // [K][2]: nb / n, na nb / n
  __shared__ double s_total;
  const long long W = 2LL * F + 1;
  if (threadIdx.x == 0) {
    double na = out_record ? 0.0 : *count;
    for (int p = 0; p < K; p++) {
      const double nb = records[p * W];
      const double n = na + nb;
      s_w[2 * p] = nb == 0.0 ? 0.0 : nb / n;
      s_w[2 * p + 1] = nb == 0.0 ? 0.0 : na * nb / n;
      na = n;
    }
    s_total = na;
  }
  __syncthreads();
  const double total = s_total;
  for (int f = threadIdx.x; f < F; f += kThreads) {
    double ma = out_record ? 0.0 : mean[f], m2a = out_record ? 0.0 : m2[f];
#pragma unroll 8
    for (int p = 0; p < K; p++) {
      const double *r = records + p * W;
      const double w1 = s_w[2 * p], w2 = s_w[2 * p + 1];
      const double mb = r[1 + f], m2b = r[1 + F + f];
      const double d = mb - ma;
      ma = ma + d * w1;
      m2a = m2a + m2b + d * d * w2;
    }
    if (out_record) {
      out_record[1 + f] = ma;
      out_record[1 + F + f] = m2a;
    } else {
      mean[f] = ma;
      m2[f] = m2a;
      // the population variance M2 / n; no samples: the identity
      shift[f] = total == 0.0 ? 0.0f : (float)ma;
      scale[f] = total == 0.0 ? 1.0f : (float)(1.0 / sqrt(m2a / total + 1e-8));
    }
  }
  __syncthreads();                              // every thread has read *count
  if (threadIdx.x == 0) {
    if (out_record) out_record[0] = total;
    else *count = total;
  }
}

__global__ void __launch_bounds__(kThreads)
obs_normalize_kernel(const float *__restrict__ x, float *__restrict__ y, long long n, int F,
                     const float *__restrict__ shift, const float *__restrict__ scale,
                     float clip) {
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n;
       i += (long long)gridDim.x * kThreads) {
    const int f = (int)(i % F);
    y[i] = obs_normalize(x[i], shift[f], scale[f], clip);
  }
}

bool shape_ok(long long rows, int F) { return rows >= 0 && F >= 1 && F <= kMaxFeatures; }

int merge(void *stream, const double *records, int K, int F, double *out_record, double *count,
          double *mean, double *m2, float *shift, float *scale) {
  const size_t smem = (size_t)K * 2 * sizeof(double);
  if (smem > 48 * 1024) return (int)cudaErrorInvalidValue;
  obs_moments_merge_kernel<<<1, kThreads, smem, as_stream(stream)>>>(
      records, K, F, out_record, count, mean, m2, shift, scale);
  return finish_launch();
}

int partials(void *stream, const float *x, long long rows, int F, double *scratch) {
  const int FT = F < kThreads ? F : kThreads;
  const dim3 grid((unsigned)n_records(rows), (unsigned)((F + FT - 1) / FT));
  obs_moments_partial_kernel<<<grid, kThreads, 0, as_stream(stream)>>>(x, rows, F, scratch);
  return finish_launch();
}

}  // namespace

WDB_API long long wdb_obs_moments_scratch_doubles(long long rows, int F) {
  if (!shape_ok(rows, F)) return -1;
  return n_records(rows) * (2LL * F + 1);
}

WDB_API int wdb_obs_moments_update(void *stream, const float *x, long long rows, int F,
                                   double *scratch, double *count, double *mean, double *m2,
                                   float *shift, float *scale) {
  if (!shape_ok(rows, F) || (rows > 0 && (!x || !scratch)) || !count || !mean || !m2 ||
      !shift || !scale)
    return (int)cudaErrorInvalidValue;
  if (rows == 0) return merge(stream, nullptr, 0, F, nullptr, count, mean, m2, shift, scale);
  const int rc = partials(stream, x, rows, F, scratch);
  if (rc != cudaSuccess) return rc;
  return merge(stream, scratch, (int)n_records(rows), F, nullptr, count, mean, m2, shift, scale);
}

WDB_API int wdb_obs_moments_batch(void *stream, const float *x, long long rows, int F,
                                  double *scratch, double *record) {
  if (!shape_ok(rows, F) || (rows > 0 && (!x || !scratch)) || !record)
    return (int)cudaErrorInvalidValue;
  if (rows == 0)
    return merge(stream, nullptr, 0, F, record, nullptr, nullptr, nullptr, nullptr, nullptr);
  const int rc = partials(stream, x, rows, F, scratch);
  if (rc != cudaSuccess) return rc;
  return merge(stream, scratch, (int)n_records(rows), F, record, nullptr, nullptr, nullptr,
               nullptr, nullptr);
}

WDB_API int wdb_obs_moments_merge(void *stream, const double *records, int n_records_in, int F,
                                  double *count, double *mean, double *m2, float *shift,
                                  float *scale) {
  if (!shape_ok(0, F) || n_records_in < 0 || n_records_in > kMaxRecords ||
      (n_records_in > 0 && !records) || !count || !mean || !m2 || !shift || !scale)
    return (int)cudaErrorInvalidValue;
  return merge(stream, records, n_records_in, F, nullptr, count, mean, m2, shift, scale);
}

WDB_API int wdb_obs_normalize(void *stream, const float *x, float *y, long long rows, int F,
                              const float *shift, const float *scale, float clip) {
  if (!shape_ok(rows, F) || !(clip > 0.0f) || !std::isfinite(clip) ||
      (rows > 0 && (!x || !y || !shift || !scale)))
    return (int)cudaErrorInvalidValue;
  const long long n = rows * F;
  if (n == 0) return cudaSuccess;
  long long blocks = (n + kThreads - 1) / kThreads;
  if (blocks > 132LL * 16) blocks = 132LL * 16;
  obs_normalize_kernel<<<(unsigned)blocks, kThreads, 0, as_stream(stream)>>>(x, y, n, F, shift,
                                                                            scale, clip);
  return finish_launch();
}
