// Seeded temperature / top-k / top-p sampling over fp32 logits rows: the draw that replaces the decode step's argmax
// (metamorph_llama.py:542) when a sequence asks for sampling. HF's warper order (TemperatureLogitsWarper ->
// TopKLogitsWarper -> TopPLogitsWarper), then a Gumbel-max draw over the kept set.
//
// One cluster of kSampleCTAs CTAs per row. Each CTA holds its slice of the row in shared memory and every pass after the
// load runs out of it: the row max, the fixed-point masses, the radix select of the top-k / top-p thresholds and the
// Gumbel argmax. CTAs combine partial maxima and histograms through distributed shared memory; there is no global
// workspace and no float atomic, so the token is a pure function of (logits bits, T, k, p, seed, counter).
//
// Rows without a usable scaled maximum never reach the draw: a row with no logit above -inf returns 0, and a row whose
// max l / T is not finite (a +inf logit, or |max l| / T overflowing fp32 at a tiny T) returns the argmax of the logits,
// lowest index among the maxima, whatever k, p and the seed are.
#include <cooperative_groups.h>
#include <math.h>
#include <mutex>

#include "common.cuh"

namespace cg = cooperative_groups;

namespace {

constexpr int kSampleCTAs = 8;          // CTAs per row (one thread-block cluster)
constexpr int kSampleThreads = 512;
constexpr int kMaxSlice = 48 * 1024;    // fp32 logits per CTA held in shared memory (192 KB)
constexpr int kBins = 2048;             // radix rounds of 11, 11 and 10 bits
constexpr int kOwn = kBins / kSampleCTAs;
constexpr float kMassScale = 1099511627776.0f;   // 2^40: mass_j = round(exp(z_j - max z) * 2^40)

constexpr size_t smem_bytes(int slice) { return (size_t)slice * 4 + (size_t)kBins * (4 + 8); }

// ---------------------------------------------------------------- Philox4x32-10 (Salmon et al., SC'11)
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += 0x9E3779B9u;
    k.y += 0xBB67AE85u;
  }
  return c;
}

// -log(u) for u = (w + 0.5) * 2^-32. The upper half goes through 1 - u = (~w + 0.5) * 2^-32, which fp32 holds to full
// relative precision, so u never rounds to 1 and the Gumbel noise stays finite.
__device__ __forceinline__ float neg_log_uniform(uint32_t w) {
  if (w < 0x80000000u) return -logf(((float)w + 0.5f) * 2.3283064365386963e-10f);
  return -log1pf(-(((float)(~w) + 0.5f) * 2.3283064365386963e-10f));
}

// order-preserving uint32 key of a float (-0 is folded into +0 before keys are taken)
__device__ __forceinline__ uint32_t f2key(float f) {
  const uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__device__ __forceinline__ unsigned long long fixed_mass(float z, float zmax) {
  if (z == zmax) return 1ull << 40;
  return (unsigned long long)__float2ull_rn(expf(z - zmax) * kMassScale);
}

__device__ __forceinline__ void better(float& best, int& bi, float v, int i) {
  if (v > best || (v == best && i < bi)) { best = v; bi = i; }
}

// (max, lowest index of the max) over the block; NaN never wins. Valid in thread 0.
__device__ __forceinline__ void block_argmax(float& best, int& bi, float* sval, int* sidx) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    better(best, bi, __shfl_xor_sync(0xffffffffu, best, o), __shfl_xor_sync(0xffffffffu, bi, o));
  if ((threadIdx.x & 31) == 0) { sval[threadIdx.x >> 5] = best; sidx[threadIdx.x >> 5] = bi; }
  __syncthreads();
  if (threadIdx.x == 0)
    for (int w = 1; w < kSampleThreads / 32; ++w) better(best, bi, sval[w], sidx[w]);
}

struct SampleShared {
  float sval[kSampleThreads / 32];
  int sidx[kSampleThreads / 32];
  float cval[2];                        // this CTA's partial (max, index) for the cluster: [0] row max, [1] draw
  int cidx[2];
  float row_max;
  int row_idx;
  uint32_t own_cnt[kOwn];               // this CTA's share of the cluster histogram (bins rank*kOwn ...)
  unsigned long long own_mass[kOwn];
  uint32_t wcnt[kSampleThreads / 32];
  unsigned long long wmass[kSampleThreads / 32];
  int pick;
  uint32_t pick_cnt;
  unsigned long long pick_mass;
};

// Combine the 8 CTAs' (cval[slot], cidx[slot]) in rank order. Every CTA gets the same answer.
__device__ __forceinline__ void cluster_argmax(cg::cluster_group& cluster, SampleShared& sh, int slot, float& best,
                                               int& bi) {
  if (threadIdx.x == 0) { sh.cval[slot] = best; sh.cidx[slot] = bi; }
  cluster.sync();
  if (threadIdx.x == 0) {
    best = -INFINITY;
    bi = 0x7fffffff;
    for (int q = 0; q < kSampleCTAs; ++q) {
      SampleShared* o = cluster.map_shared_rank(&sh, q);
      better(best, bi, o->cval[slot], o->cidx[slot]);
    }
    sh.row_max = best;
    sh.row_idx = bi;
  }
  __syncthreads();
  best = sh.row_max;
  bi = sh.row_idx;
}

// MSB-first radix select over the keys >= kmin of the row. Returns the key t of the lowest kept value:
//   by_mass = false: the k-th largest value, so {z >= t} = {z : count(z_j > z) < k} (ties at t kept);
//   by_mass = true : the lowest value v with mass(z_j > v, z_j >= kmin) < p * mass(z_j >= kmin).
// Each round histograms (count, fixed-point mass) of the keys under the current prefix, sums the 8 CTAs' histograms
// through DSMEM (CTA q owns bins [q*kOwn, (q+1)*kOwn)), gathers the full sum back into its own histogram and picks the
// lowest non-empty bin whose "strictly above" count / mass still passes the test.
__device__ uint32_t radix_select(cg::cluster_group& cluster, SampleShared& sh, const float* zs, int n, float zmax,
                                 uint32_t kmin, bool by_mass, uint32_t k, float p, uint32_t* hcnt,
                                 unsigned long long* hmass) {
  const int tid = threadIdx.x, rank = (int)cluster.block_rank();
  uint32_t prefix = 0, above_cnt = 0;
  unsigned long long above_mass = 0;
  double thresh = 0.0;
  int done_bits = 0;
  for (int round = 0; round < 3; ++round) {
    const int bits = round < 2 ? 11 : 10, nb = 1 << bits, shift = 32 - done_bits - bits;
    for (int b = tid; b < kBins; b += kSampleThreads) { hcnt[b] = 0; hmass[b] = 0; }
    __syncthreads();
    for (int j = tid; j < n; j += kSampleThreads) {
      const float z = zs[j];
      const uint32_t key = f2key(z);
      if (key < kmin || (done_bits > 0 && (key >> (32 - done_bits)) != prefix)) continue;
      const uint32_t d = (key >> shift) & (nb - 1);
      atomicAdd(&hcnt[d], 1u);
      if (by_mass) atomicAdd(&hmass[d], fixed_mass(z, zmax));
    }
    cluster.sync();                                      // every CTA's histogram is complete
    if (tid < kOwn) {
      const int b = rank * kOwn + tid;
      uint32_t c = 0;
      unsigned long long m = 0;
      for (int q = 0; q < kSampleCTAs; ++q) {
        c += cluster.map_shared_rank(hcnt, q)[b];
        m += cluster.map_shared_rank(hmass, q)[b];
      }
      sh.own_cnt[tid] = c;
      sh.own_mass[tid] = m;
    }
    cluster.sync();                                      // every owner has summed its bins; histograms are free again
    for (int b = tid; b < kBins; b += kSampleThreads) {
      SampleShared* o = cluster.map_shared_rank(&sh, b / kOwn);
      hcnt[b] = o->own_cnt[b % kOwn];
      hmass[b] = o->own_mass[b % kOwn];
    }
    if (tid == 0) sh.pick = 0x7fffffff;
    __syncthreads();
    // suffix sums: thread t owns bins [t*per, t*per + per); "above" = all bins of higher digit
    const int per = nb / kSampleThreads;
    uint32_t tc = 0;
    unsigned long long tm = 0;
    for (int i = 0; i < per; ++i) { tc += hcnt[tid * per + i]; tm += hmass[tid * per + i]; }
    const int lane = tid & 31, warp = tid >> 5;
    uint32_t sc = tc;
    unsigned long long sm = tm;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t c2 = __shfl_down_sync(0xffffffffu, sc, o);
      const unsigned long long m2 = __shfl_down_sync(0xffffffffu, sm, o);
      if (lane + o < 32) { sc += c2; sm += m2; }
    }
    if (lane == 0) { sh.wcnt[warp] = sc; sh.wmass[warp] = sm; }
    __syncthreads();
    uint32_t ac = above_cnt + (sc - tc);
    unsigned long long am = above_mass + (sm - tm);
    for (int w = warp + 1; w < kSampleThreads / 32; ++w) { ac += sh.wcnt[w]; am += sh.wmass[w]; }
    if (round == 0 && by_mass) {
      unsigned long long total = 0;
      for (int w = 0; w < kSampleThreads / 32; ++w) total += sh.wmass[w];
      thresh = (double)p * (double)total;
    }
    int cand = 0x7fffffff;
    uint32_t cand_c = 0;
    unsigned long long cand_m = 0;
    for (int i = per - 1; i >= 0; --i) {
      const int b = tid * per + i;
      const bool pass = by_mass ? (double)am < thresh : ac < k;
      if (hcnt[b] > 0 && pass) { cand = b; cand_c = ac; cand_m = am; }
      ac += hcnt[b];
      am += hmass[b];
    }
    if (cand != 0x7fffffff) atomicMin(&sh.pick, cand);
    __syncthreads();
    if (cand != 0x7fffffff && cand == sh.pick) { sh.pick_cnt = cand_c; sh.pick_mass = cand_m; }
    __syncthreads();
    prefix = (prefix << bits) | (uint32_t)sh.pick;
    above_cnt = sh.pick_cnt;
    above_mass = sh.pick_mass;
    done_bits += bits;
    __syncthreads();
  }
  return prefix;
}

__global__ void __cluster_dims__(kSampleCTAs, 1, 1) __launch_bounds__(kSampleThreads, 1)
sample_rows_kernel(const float* __restrict__ logits, long long ld, int V, int S, const float* __restrict__ temperature,
                   const int* __restrict__ top_k, const float* __restrict__ top_p,
                   const unsigned long long* __restrict__ seed, const int* __restrict__ counter, int* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char dyn[];
  __shared__ SampleShared sh;
  float* zs = reinterpret_cast<float*>(dyn);
  uint32_t* hcnt = reinterpret_cast<uint32_t*>(zs + S);
  unsigned long long* hmass = reinterpret_cast<unsigned long long*>(hcnt + kBins);
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank(), tid = threadIdx.x;
  const long long r = blockIdx.x / kSampleCTAs;
  const int j0 = rank * S;
  const int n = max(0, min(S, V - j0));
  const float* x = logits + r * ld + j0;

  // load the slice; the argmax of the raw logits is the greedy token and gives max z
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int j = tid; j < n; j += kSampleThreads) {
    const float v = x[j];
    zs[j] = v;
    if (v > best) { best = v; bi = j0 + j; }
  }
  block_argmax(best, bi, sh.sval, sh.sidx);
  cluster_argmax(cluster, sh, 0, best, bi);

  const float T = temperature[r];
  const bool greedy = !(T > 0.f);                        // T <= 0 or NaN
  const float zmax = best / T;
  // Greedy, no logit above -inf, or max z = +-inf: a +inf logit, or a temperature so small that the divide overflows.
  // Then z - max z is NaN or every scaled value collapses onto +-inf, and the row returns the limit T -> 0 of the draw:
  // the argmax of the logits, lowest index among the maxima (bi is unset only when no logit is above -inf).
  if (greedy || !(best > -INFINITY) || isinf(zmax)) {
    if (rank == 0 && tid == 0) out[r] = bi != 0x7fffffff ? bi : 0;
    cluster.sync();                                      // keep this CTA's shared memory alive for the readers
    return;
  }
  for (int j = tid; j < n; j += kSampleThreads) {
    const float v = zs[j];
    float z = isnan(v) ? -INFINITY : v / T;
    zs[j] = z == 0.f ? 0.f : z;                          // -0 -> +0: keys then order by value
  }
  __syncthreads();

  const int k = top_k[r];
  const float p = top_p[r];
  uint32_t t = 0;                                        // keep keys >= t
  if (k > 0 && k < V) t = radix_select(cluster, sh, zs, n, zmax, 0, false, (uint32_t)k, 0.f, hcnt, hmass);
  if (p <= 0.f) t = f2key(zmax == 0.f ? 0.f : zmax);
  else if (p < 1.f) t = radix_select(cluster, sh, zs, n, zmax, t, true, 0, p, hcnt, hmass);

  // Gumbel-max over the kept set: u_i from word (i & 3) of Philox4x32-10(counter (i >> 2, c, 0, 0), key (s_lo, s_hi))
  const unsigned long long s = seed[r];
  const uint2 key = make_uint2((uint32_t)s, (uint32_t)(s >> 32));
  const uint32_t c = (uint32_t)counter[r];
  best = -INFINITY;
  bi = 0x7fffffff;
  for (int g = tid; g * 4 < n; g += kSampleThreads) {
    bool any = false;
#pragma unroll
    for (int e = 0; e < 4; ++e) any |= g * 4 + e < n && f2key(zs[g * 4 + e]) >= t;
    if (!any) continue;
    const uint4 w = philox4x32_10(make_uint4((uint32_t)((j0 + g * 4) >> 2), c, 0u, 0u), key);
    const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int j = g * 4 + e;
      if (j >= n) break;
      const float z = zs[j];
      if (f2key(z) < t) continue;
      better(best, bi, z - logf(neg_log_uniform(ws[e])), j0 + j);
    }
  }
  block_argmax(best, bi, sh.sval, sh.sidx);
  cluster_argmax(cluster, sh, 1, best, bi);
  if (rank == 0 && tid == 0) out[r] = bi != 0x7fffffff ? bi : 0;
  cluster.sync();
}

// ---------------------------------------------------------------- log-probabilities of the emitted token
// logprob(i) = l_i - m - ln S over the raw logits (NaN read as -inf), m = max l, S = sum_j exp(l_j - m), rounded once to
// fp32. Each term is expf(d_hi) * (1 + d_lo) with d = l_j - m split into fp32 d_hi and the fp64 remainder d_lo, so the
// term carries expf's 2 ulp and nothing of the fp32 rounding of d; S is summed in fp64 in a fixed order (per thread
// j = tid, tid + 512, ..., the warp tree, warps in order, CTAs in rank order) that depends on V alone.
// The top-n list orders (l, index) by value descending, lowest index first among ties: mm_argmax_rows' order.
constexpr int kTopMax = 20;

struct LogprobShared {
  float sval[kSampleThreads / 32];
  int sidx[kSampleThreads / 32];
  float wmax[kSampleThreads / 32];
  int wcnt[kSampleThreads / 32];
  double wsum[kSampleThreads / 32];
  float cmax;                           // this CTA's partials for the cluster: max, count of +inf, sum of exp(l - m)
  int ccnt;
  double csum;
  float top_v[kTopMax];                 // this CTA's top-n, in order; index 0x7fffffff = no entry
  int top_i[kTopMax];
  float pick_v;
  int pick_i;
  float row_max;
};

// (v, i) comes strictly after (pv, pi) in the top-n order
__device__ __forceinline__ bool after(float v, int i, float pv, int pi) { return v < pv || (v == pv && i > pi); }

// mode 0: a distribution (lnS = ln S); 1: max is +inf (lnS = ln c, c = count of +inf); 2: no logit above -inf
__device__ __forceinline__ float logprob_of(float v, float m, double lnS, int mode) {
  if (mode == 2) return __int_as_float(0x7fffffff);
  if (mode == 1) return v == INFINITY ? (float)(-lnS) : -INFINITY;
  return (float)(((double)v - (double)m) - lnS);
}

__global__ void __cluster_dims__(kSampleCTAs, 1, 1) __launch_bounds__(kSampleThreads, 1)
decode_logprobs_kernel(const float* __restrict__ logits, long long ld, int V, int S,
                       const int* __restrict__ append_kind, const int* __restrict__ token,
                       const int* __restrict__ n_ids, const int* __restrict__ n_top, int max_ids,
                       float* __restrict__ lp_out, int* __restrict__ top_ids, float* __restrict__ top_lp) {
  extern __shared__ __align__(16) unsigned char dyn[];
  __shared__ LogprobShared sh;
  float* zs = reinterpret_cast<float*>(dyn);
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank(), tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long r = blockIdx.x / kSampleCTAs;
  // every CTA of the cluster reads the same gate, so a skipped row leaves without touching the cluster
  const int slot = n_ids[r] - 1, nt = n_top[r];
  if (append_kind[r] != 0 || nt < 0 || slot < 0 || slot >= max_ids) return;
  const int ntop = min(nt, kTopMax);
  const int j0 = rank * S;
  const int n = max(0, min(S, V - j0));
  const float* x = logits + r * ld + j0;

  // load the slice (NaN -> -inf); the thread's first entry in the top-n order, its max and its count of +inf
  float cv = -INFINITY;
  int ci = 0x7fffffff, cnt = 0;
  for (int j = tid; j < n; j += kSampleThreads) {
    float v = x[j];
    if (isnan(v)) v = -INFINITY;
    zs[j] = v;
    better(cv, ci, v, j0 + j);
    cnt += v == INFINITY;
  }
  float mx = cv;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  if (lane == 0) { sh.wmax[warp] = mx; sh.wcnt[warp] = cnt; }
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < kSampleThreads / 32; ++w) { mx = fmaxf(mx, sh.wmax[w]); cnt += sh.wcnt[w]; }
    sh.cmax = mx;
    sh.ccnt = cnt;
  }
  cluster.sync();                                        // every CTA's max and count are published
  if (tid == 0) {
    float m = -INFINITY;
    for (int q = 0; q < kSampleCTAs; ++q) m = fmaxf(m, cluster.map_shared_rank(&sh, q)->cmax);
    sh.row_max = m;
  }
  __syncthreads();
  const float m = sh.row_max;

  // S over the slice, fp64 (only a finite max has terms; the special rows need none)
  double s = 0.0;
  if (m > -INFINITY && m < INFINITY) {
    for (int j = tid; j < n; j += kSampleThreads) {
      const double d = (double)zs[j] - (double)m;        // -inf for a -inf logit
      if (d > -110.0) {                                  // below, expf(d) < 2^-158: the term rounds to 0
        const float dh = (float)d;
        s += (double)expf(dh) * (1.0 + (d - (double)dh));
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) sh.wsum[warp] = s;

  // this CTA's top-n: each thread holds its first entry after the last pick; only the pick's owner looks further
  for (int k = 0; k < ntop; ++k) {
    float bv = cv;
    int bj = ci;
    block_argmax(bv, bj, sh.sval, sh.sidx);
    if (tid == 0) { sh.top_v[k] = bv; sh.top_i[k] = bj; sh.pick_v = bv; sh.pick_i = bj; }
    __syncthreads();
    const float pv = sh.pick_v;
    const int pi = sh.pick_i;
    if (pi != 0x7fffffff && ci == pi) {
      cv = -INFINITY;
      ci = 0x7fffffff;
      for (int j = tid; j < n; j += kSampleThreads)
        if (after(zs[j], j0 + j, pv, pi)) better(cv, ci, zs[j], j0 + j);
    }
  }
  __syncthreads();
  if (tid == 0) {
    s = 0.0;
    for (int w = 0; w < kSampleThreads / 32; ++w) s += sh.wsum[w];
    sh.csum = s;
  }
  cluster.sync();                                        // every CTA's sum and top-n are published

  if (rank == 0 && tid == 0) {
    int mode = 0, c = 0;
    double sum = 0.0;
    for (int q = 0; q < kSampleCTAs; ++q) {
      const LogprobShared* o = cluster.map_shared_rank(&sh, q);
      sum += o->csum;
      c += o->ccnt;
    }
    double lnS = 0.0;
    if (!(m > -INFINITY)) mode = 2;
    else if (m == INFINITY) { mode = 1; lnS = log((double)c); }
    else lnS = log(sum);
    const long long o = r * max_ids + slot;
    const int t = token[r];
    float vt = __int_as_float(0x7fffffff);               // a token outside [0, V) reports NaN
    if (t >= 0 && t < V) {
      vt = logits[r * ld + t];
      vt = logprob_of(isnan(vt) ? -INFINITY : vt, m, lnS, mode);
    }
    lp_out[o] = vt;
    // merge the CTAs' sorted lists: each step takes the first head in the order
    int head[kSampleCTAs];
#pragma unroll
    for (int q = 0; q < kSampleCTAs; ++q) head[q] = 0;
    for (int k = 0; k < ntop; ++k) {
      float bv = -INFINITY;
      int bj = 0x7fffffff, bq = -1;
#pragma unroll
      for (int q = 0; q < kSampleCTAs; ++q) {
        const LogprobShared* p = cluster.map_shared_rank(&sh, q);
        if (head[q] < ntop && p->top_i[head[q]] != 0x7fffffff) {
          const float v = p->top_v[head[q]];
          const int i = p->top_i[head[q]];
          if (v > bv || (v == bv && i < bj)) { bv = v; bj = i; bq = q; }
        }
      }
      if (bq >= 0) {
#pragma unroll
        for (int q = 0; q < kSampleCTAs; ++q) head[q] += q == bq;
      }
      top_ids[o * kTopMax + k] = bq >= 0 ? bj : -1;      // fewer than n entries (V < n): id -1, logprob -inf
      top_lp[o * kTopMax + k] = bq >= 0 ? logprob_of(bv, m, lnS, mode) : -INFINITY;
    }
  }
  cluster.sync();                                        // keep every CTA's shared memory alive for rank 0
}

}  // namespace

MM_API int mm_sample_rows(const float* logits, long long ld, long long R, int V, const float* temperature,
                          const int* top_k, const float* top_p, const unsigned long long* seed, const int* counter,
                          int* out, cudaStream_t stream) {
  MM_CHECK_ARG(R > 0 && V > 0 && ld >= V, "mm_sample_rows: bad shape (need R>0, V>0, ld>=V)");
  MM_CHECK_ARG(R <= 0x7fffffffll / kSampleCTAs, "mm_sample_rows: too many rows");
  const int per = (V + kSampleCTAs - 1) / kSampleCTAs;
  const int S = (per + 3) / 4 * 4;                       // multiple of 4: a Philox block never straddles two CTAs
  MM_CHECK_ARG(S <= kMaxSlice, "mm_sample_rows: V=%d exceeds the shared-memory budget (V <= %d)", V,
               kSampleCTAs * kMaxSlice);
  MM_CHECK_ARG(logits && temperature && top_k && top_p && seed && counter && out, "mm_sample_rows: null pointer");
  static std::once_flag once;
  static cudaError_t attr_err = cudaSuccess;
  std::call_once(once, [] {
    attr_err = cudaFuncSetAttribute(sample_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)smem_bytes(kMaxSlice));
  });
  MM_CHECK_CUDA(attr_err);
  sample_rows_kernel<<<(unsigned)(R * kSampleCTAs), kSampleThreads, smem_bytes(S), stream>>>(
      logits, ld, V, S, temperature, top_k, top_p, seed, counter, out);
  MM_CHECK_LAUNCH();
  return MM_OK;
}

MM_API int mm_decode_logprobs(const float* logits, long long ld, long long R, int V, const int* append_kind,
                              const int* token, const int* n_ids, const int* n_top, int max_ids, float* lp_out,
                              int* top_ids, float* top_lp, cudaStream_t stream) {
  MM_CHECK_ARG(R > 0 && V > 0 && ld >= V && max_ids > 0,
               "mm_decode_logprobs: bad shape (need R>0, V>0, ld>=V, max_ids>0)");
  MM_CHECK_ARG(R <= 0x7fffffffll / kSampleCTAs, "mm_decode_logprobs: too many rows");
  const int S = ((V + kSampleCTAs - 1) / kSampleCTAs + 3) / 4 * 4;   // the slice rule of mm_sample_rows
  MM_CHECK_ARG(S <= kMaxSlice, "mm_decode_logprobs: V=%d exceeds the shared-memory budget (V <= %d)", V,
               kSampleCTAs * kMaxSlice);
  MM_CHECK_ARG(logits && append_kind && token && n_ids && n_top && lp_out && top_ids && top_lp,
               "mm_decode_logprobs: null pointer");
  static std::once_flag once;
  static cudaError_t attr_err = cudaSuccess;
  std::call_once(once, [] {
    attr_err = cudaFuncSetAttribute(decode_logprobs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    kMaxSlice * 4);
  });
  MM_CHECK_CUDA(attr_err);
  decode_logprobs_kernel<<<(unsigned)(R * kSampleCTAs), kSampleThreads, (size_t)S * 4, stream>>>(
      logits, ld, V, S, append_kind, token, n_ids, n_top, max_ids, lp_out, top_ids, top_lp);
  MM_CHECK_LAUNCH();
  return MM_OK;
}
