// Token sampling on the device: one token per row of bf16 logits, greedy or temperature / top-k / top-p / min-p, drawn from a
// counter-based Philox4x32-10 stream, so a decode step captured in a CUDA graph can pick its next token without the host.
//
// The contract (ops.sample_tokens states it in full): greedy = the lowest index among the maximal logits. Otherwise
// p_i = exp((l_i - l_max) / T), and the filters keep, in turn, every token at least as large as the k-th largest logit (top-k), the
// largest upper set of that set whose mass reaches top_p of its mass (top-p: the tie group that crosses is kept whole), and every
// l_i >= l_max + T·ln(min_p) (min-p). Each filter keeps an upper set of the logit order, so the keep-set is {key >= t*, l >= thr}.
// The draw is the inverse CDF in vocabulary order: with target = u·mass(kept), the first kept index whose inclusive prefix mass
// exceeds target. u = ((x0 >> 8) + 0.5)·2^-24 with x0 the first word of Philox4x32-10 (key = the row's 64-bit seed, counter =
// (position, 0, 0, 0)).
//
// Determinism: a token's mass is p_i in fp64 (p_max = 1) rounded to a 2^-40 fixed-point integer, and every sum -- histogram bins,
// the top-p mass, the prefix of the draw -- is an integer sum, exact in any order. So the same inputs give the same token on every
// run, whatever order the shared-memory atomics land in.
//
// Thresholds by radix select over the 16-bit order key of bf16 (sign-flipped bits): one 256-bin histogram over the high byte, then
// one over the low byte of the chosen high bin, whose bins are single bf16 values (tie groups).
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kSampThreads = 512;
constexpr int kSampWarps = kSampThreads / 32;
constexpr int kTile = kSampThreads * 8;         // one sweep of the CTA: 8 consecutive logits per thread, one 16-byte load if aligned
constexpr double kMassUnit = 1099511627776.0;  // 2^40: fixed-point scale of a token's mass p_i in [0, 1]

struct SampleParams {
  const uint16_t* logits;  // bf16 bits, row b at b·ld
  int64_t ld;
  int V, top_k;
  float temperature, top_p, minp_off;  // minp_off = T·ln(min_p) (-inf when off)
  double inv_t;                        // 1 / T
  bool vec;                            // rows 16-byte aligned: vector loads
  const int64_t* seeds;
  const int* positions;
  int64_t* out;
  // bookkeeping (all null or none)
  int64_t* history;
  int* n_out;
  uint8_t* active;
  const int* prompt_len;
  int max_new, max_seq_len;
  int64_t eos;
};

// order key: larger key = larger value; -0 is folded onto +0 so that equal values have equal keys
__device__ __forceinline__ uint32_t order_key(uint32_t bits) {
  bits = bits == 0x8000u ? 0u : bits;
  return (bits & 0x8000u) ? (~bits & 0xFFFFu) : (bits | 0x8000u);
}

__device__ __forceinline__ float key_value(uint32_t key) {
  const uint32_t bits = (key & 0x8000u) ? (key & 0x7FFFu) : (~key & 0xFFFFu);
  return __uint_as_float(bits << 16);
}

// keys of logits i0 .. i0 + 7 of a row; n = how many of them are < V
__device__ __forceinline__ int load8(const SampleParams& p, const uint16_t* row, int i0, uint32_t (&k)[8]) {
  const int n = min(8, p.V - i0);
  if (p.vec && n == 8) {
    const uint4 v = *reinterpret_cast<const uint4*>(row + i0);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      k[2 * j] = order_key(w[j] & 0xFFFFu);
      k[2 * j + 1] = order_key(w[j] >> 16);
    }
  } else {
#pragma unroll
    for (int j = 0; j < 8; ++j) k[j] = j < n ? order_key(row[i0 + j]) : 0u;
  }
  return n;
}

__device__ __forceinline__ uint64_t warp_incl_scan(uint64_t x) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint64_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  return x;
}

// Inclusive prefix over the CTA in thread order; `total` = the sum over all threads. s_w: kSampWarps words of shared memory.
__device__ __forceinline__ uint64_t block_incl_scan(uint64_t v, uint64_t* s_w, uint64_t& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint64_t x = warp_incl_scan(v);
  if (lane == 31) s_w[warp] = x;
  __syncthreads();
  uint64_t off = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < kSampWarps; ++w) {
    const uint64_t t = s_w[w];
    off += w < warp ? t : 0;
    tot += t;
  }
  __syncthreads();  // s_w is reused by the next call
  total = tot;
  return x + off;
}

__device__ __forceinline__ uint64_t block_max(uint64_t v, uint64_t* s_w) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max(v, (uint64_t)__shfl_xor_sync(0xffffffffu, v, o));
  if (lane == 0) s_w[warp] = v;
  __syncthreads();
  uint64_t m = 0;
#pragma unroll
  for (int w = 0; w < kSampWarps; ++w) m = max(m, s_w[w]);
  __syncthreads();
  return m;
}

// Run by one full warp over a 256-bin histogram h: going down from bin 255 to bin lo, the first bin whose inclusive cumulative sum
// (plus base) reaches goal, and in *above the cumulative sum (plus base) of the bins above it. Returns -1 (and the whole sum) if no
// bin reaches it. Lane j owns bins 255 - 8j down to 248 - 8j.
__device__ int warp_find_desc(const uint64_t* h, int lo, uint64_t base, double goal, uint64_t* above) {
  const int lane = threadIdx.x & 31;
  uint64_t own = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int bin = 255 - 8 * lane - j;
    own += bin >= lo ? h[bin] : 0;
  }
  const uint64_t incl = warp_incl_scan(own) + base;
  const unsigned hit = __ballot_sync(0xffffffffu, (double)incl >= goal);
  if (hit == 0) {
    *above = __shfl_sync(0xffffffffu, incl, 31);
    return -1;
  }
  const int src = __ffs(hit) - 1;
  int found = -1;
  uint64_t c = incl - own;
  if (lane == src) {
    for (int j = 0; j < 8; ++j) {
      const int bin = 255 - 8 * lane - j;
      if (bin < lo) break;
      if ((double)(c + h[bin]) >= goal) {
        found = bin;
        break;
      }
      c += h[bin];
    }
  }
  *above = __shfl_sync(0xffffffffu, c, src);
  return __shfl_sync(0xffffffffu, found, src);
}

__device__ __forceinline__ uint4 philox4x32_10(uint32_t k0, uint32_t k1, uint4 c) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r > 0) {
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
    const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
  }
  return c;
}

// fixed-point mass of a key: p = exp((l - l_max)·(1/T)) in fp64, so that the fixed-point rounding (2^-41) and not exp's error bounds
// how far a mass is from exact
__device__ __forceinline__ uint64_t key_mass(uint32_t key, const double& lmax_d, const double& inv_t) {
  return __double2ull_rn(exp(((double)key_value(key) - lmax_d) * inv_t) * kMassUnit);
}

// The row's maximum key, lowest index among equals: (key, ~index) packed so that one max picks both.
// k: the caller's key buffer (one buffer for every pass keeps the sampler's register allocation).
__device__ __forceinline__ uint64_t row_best(const SampleParams& p, const uint16_t* row, uint64_t* s_w, uint32_t (&k)[8]) {
  const int tid = threadIdx.x, V = p.V;
  uint64_t best = 0;
  for (int i0 = tid * 8; i0 < V; i0 += kTile) {
    const int n = load8(p, row, i0, k);
    for (int j = 0; j < n; ++j) best = max(best, ((uint64_t)k[j] << 32) | (0xFFFFFFFFu - (uint32_t)(i0 + j)));
  }
  return block_max(best, s_w);
}

// The top-k / top-p threshold key t*: the keep-set of temperature > 0 sampling is {key >= t*, l >= l_max + T·ln(min_p)}.
// High-byte histogram of counts and masses, then one or two low-byte histograms of a single high bin. 0 = no threshold.
__device__ __forceinline__ uint32_t keep_threshold(const SampleParams& p, const uint16_t* row, const double& lmax_d, const double& inv_t,
                                                   uint32_t (&k)[8], uint64_t (&s_hc)[256], uint64_t (&s_hm)[256],
                                                   uint64_t (&s_lc)[256], uint64_t (&s_lm)[256], int (&s_bin)[2], uint64_t& s_above,
                                                   double& s_need) {
  const int tid = threadIdx.x, V = p.V;
  auto mass = [&](uint32_t key) -> uint64_t { return key_mass(key, lmax_d, inv_t); };
  const bool use_k = p.top_k > 0 && p.top_k < V, use_p = p.top_p < 1.f;
  uint32_t t_key = 0;  // keep key >= t_key (top-k and top-p)
  if (use_k || use_p) {
    for (int i = tid; i < 256; i += kSampThreads) s_hc[i] = s_hm[i] = 0;
    __syncthreads();
    for (int i0 = tid * 8; i0 < V; i0 += kTile) {
      const int n = load8(p, row, i0, k);
      for (int j = 0; j < n; ++j) {
        atomicAdd((unsigned long long*)&s_hc[k[j] >> 8], 1ull);
        if (use_p) atomicAdd((unsigned long long*)&s_hm[k[j] >> 8], (unsigned long long)mass(k[j]));
      }
    }
    __syncthreads();
    int hb = 0, lb = 0;  // top-k threshold key hb·256 + lb (0: everything)
    if (use_k) {
      // high bin holding the k-th largest key, then its low byte among that bin's keys
      if (tid < 32) {
        uint64_t above;
        const int bin = warp_find_desc(s_hc, 0, 0, (double)p.top_k, &above);
        if (tid == 0) {
          s_bin[0] = bin;
          s_above = above;
        }
      }
      for (int i = tid; i < 256; i += kSampThreads) s_lc[i] = s_lm[i] = 0;
      __syncthreads();
      hb = s_bin[0];
      for (int i0 = tid * 8; i0 < V; i0 += kTile) {
        const int n = load8(p, row, i0, k);
        for (int j = 0; j < n; ++j) {
          if ((int)(k[j] >> 8) != hb) continue;
          atomicAdd((unsigned long long*)&s_lc[k[j] & 255u], 1ull);
          if (use_p) atomicAdd((unsigned long long*)&s_lm[k[j] & 255u], (unsigned long long)mass(k[j]));
        }
      }
      __syncthreads();
      if (tid < 32) {
        uint64_t above;
        const int bin = warp_find_desc(s_lc, 0, s_above, (double)p.top_k, &above);
        if (tid == 0) s_bin[1] = bin;
      }
      __syncthreads();
      lb = s_bin[1];
      t_key = (uint32_t)(hb << 8 | lb);
    }
    if (use_p) {
      // S = the top-k set: every high bin above hb, and the low bins >= lb of bin hb (all of bin hb without top-k)
      if (tid < 32) {
        uint64_t above_hb, in_hb = 0;
        warp_find_desc(s_hm, hb + 1, 0, INFINITY, &above_hb);  // no bin reaches +inf: the sum of the bins above hb
        if (use_k) {
          uint64_t t;
          warp_find_desc(s_lm, lb, 0, INFINITY, &t);
          in_hb = t;
        } else {
          in_hb = s_hm[hb];
        }
        const double need = (double)p.top_p * (double)(above_hb + in_hb);
        uint64_t above;
        int bin = warp_find_desc(s_hm, hb + 1, 0, need, &above);
        if (bin < 0) bin = hb;  // the crossing is in the boundary bin; `above` is then the mass of the bins above it
        if (tid == 0) {
          s_bin[0] = bin;
          s_above = above;
          s_need = need;
        }
      }
      __syncthreads();
      const int hp = s_bin[0];
      const bool reuse = use_k && hp == hb;  // the low histogram of bin hb, restricted to S, is already there
      if (!reuse) {
        for (int i = tid; i < 256; i += kSampThreads) s_lm[i] = 0;
        __syncthreads();
        for (int i0 = tid * 8; i0 < V; i0 += kTile) {
          const int n = load8(p, row, i0, k);
          for (int j = 0; j < n; ++j)
            if ((int)(k[j] >> 8) == hp) atomicAdd((unsigned long long*)&s_lm[k[j] & 255u], (unsigned long long)mass(k[j]));
        }
        __syncthreads();
      }
      if (tid < 32) {
        uint64_t above;
        const int bin = warp_find_desc(s_lm, reuse ? lb : 0, s_above, s_need, &above);
        if (tid == 0) s_bin[1] = bin < 0 ? (reuse ? lb : 0) : bin;  // unreachable: need <= mass(S)
      }
      __syncthreads();
      t_key = max(t_key, (uint32_t)(hp << 8 | s_bin[1]));
    }
  }
  return t_key;
}

// u·M = (2r + 1)·M / 2^25 with r the top 24 bits of x0, in integers (M < 2^63, so the product needs 88 bits)
__device__ __forceinline__ uint64_t draw_target(uint32_t x0, uint64_t M) {
  const uint64_t a = 2ull * (x0 >> 8) + 1ull;
  return (__umul64hi(a, M) << 39) | ((a * M) >> 25);
}

// Index-order inverse CDF, one tile of kTile entries at a time: the first index whose inclusive prefix of weights exceeds target, or
// -1 if none does. weight(i0, n, m8) fills the weights of entries i0 .. i0 + 7 (n of them < V). s_tok: one shared word.
template <class W>
__device__ __forceinline__ int64_t inverse_cdf(const int& V, const uint64_t& target, W weight, uint64_t* s_w, int64_t* s_tok) {
  const int tid = threadIdx.x;
  if (tid == 0) *s_tok = -1;
  uint64_t carry = 0;
  for (int base = 0; base < V; base += kTile) {
    const int i0 = base + tid * 8;
    uint64_t m8[8], sum = 0;
    weight(i0, m8);
#pragma unroll
    for (int j = 0; j < 8; ++j) sum += m8[j];
    uint64_t tile;
    const uint64_t incl = block_incl_scan(sum, s_w, tile) + carry;
    if (incl - sum <= target && target < incl) {
      uint64_t c = incl - sum;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        c += m8[j];
        if (c > target) {
          *s_tok = i0 + j;
          break;
        }
      }
    }
    __syncthreads();
    if (*s_tok >= 0) break;
    carry += tile;
  }
  return *s_tok;
}

// One CTA per row. Passes over the row (the first from HBM, the rest mostly from L2): the maximum; with top-k or top-p a high-byte
// histogram of counts and masses and one or two low-byte histograms of a single high bin; the kept mass; the index-order draw.
__global__ void __launch_bounds__(kSampThreads) sample_tokens_kernel(const SampleParams p) {
  __shared__ uint64_t s_w[kSampWarps];
  __shared__ uint64_t s_hc[256], s_hm[256], s_lc[256], s_lm[256];  // counts / masses: high byte, low byte of one high bin
  __shared__ int s_bin[2];
  __shared__ uint64_t s_above;
  __shared__ double s_need;
  __shared__ int64_t s_tok;

  const int b = blockIdx.x, tid = threadIdx.x;
  if (p.active != nullptr && p.active[b] == 0) return;  // a finished row writes nothing
  const uint16_t* row = p.logits + (int64_t)b * p.ld;
  const int V = p.V;
  uint32_t k[8];

  uint64_t best = row_best(p, row, s_w, k);
  const uint32_t kmax = (uint32_t)(best >> 32);
  int64_t token = (int64_t)(0xFFFFFFFFu - (uint32_t)best);

  if (p.temperature > 0.f) {
    const float lmax = key_value(kmax);
    const double lmax_d = lmax, inv_t = p.inv_t;
    const float thr = lmax + p.minp_off;  // min-p: l >= l_max + T·ln(min_p)
    const uint32_t t_key = keep_threshold(p, row, lmax_d, inv_t, k, s_hc, s_hm, s_lc, s_lm, s_bin, s_above, s_need);
    auto kept_mass = [&](uint32_t key) -> uint64_t { return key >= t_key && key_value(key) >= thr ? key_mass(key, lmax_d, inv_t) : 0; };

    // kept mass, then the target
    uint64_t own = 0;
    for (int i0 = tid * 8; i0 < V; i0 += kTile) {
      const int n = load8(p, row, i0, k);
      for (int j = 0; j < n; ++j) own += kept_mass(k[j]);
    }
    uint64_t M;
    block_incl_scan(own, s_w, M);
    const uint64_t seed = (uint64_t)p.seeds[b];
    const uint4 x = philox4x32_10((uint32_t)seed, (uint32_t)(seed >> 32), make_uint4((uint32_t)p.positions[b], 0u, 0u, 0u));
    const uint64_t target = draw_target(x.x, M);

    // index-order draw: the thread whose 8 logits straddle target finds the index
    const int64_t tok = inverse_cdf(V, target, [&](int i0, uint64_t (&m8)[8]) {
      const int n = i0 < V ? load8(p, row, i0, k) : 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) m8[j] = j < n ? kept_mass(k[j]) : 0;
    }, s_w, &s_tok);
    // target < M, so the draw always lands; the argmax (always kept) stands in for the unreachable fallback
    if (tok >= 0) token = tok;
  }

  if (tid != 0) return;
  p.out[b] = token;
  if (p.history != nullptr) {
    const int n = p.n_out[b];
    p.history[(int64_t)b * p.max_new + n] = token;
    p.n_out[b] = n + 1;
    if (n + 1 >= p.max_new || p.prompt_len[b] + n + 1 >= p.max_seq_len || token == p.eos) p.active[b] = 0;
  }
}

// ------------------------------------------------------------------------------------------------------ speculative accept
// The round of ops.spec_accept: P_i / Q_i are the filtered target / draft distributions of query i, each normalised to 2^-40 fixed
// point by one correctly rounded fp64 division per token. d_i is accepted iff (2r + 1)·Q_i[d_i] < 2^25·P_i[d_i] (r from Philox
// counter (L + i, 1, 0, 0)); at the first rejection y is drawn from max(0, P_i - Q_i), after k acceptances from P_{k+1}, by the
// index-order inverse CDF with counter (L + i, 2, 0, 0). Greedy: accept iff d_i is the argmax of p_i, y = that argmax.
struct SpecParams {
  SampleParams tp, dp;  // target rows [B·(k+1), V] (row b·(k+1) + t) and draft rows [k·B, V] (row i·B + b); knobs in both
  int k, B;
  const int64_t* tokens;  // [B, k+1]: the pending token x, then d_1 .. d_k
  const int* lo_q;        // [B, k+1]: each verify query's document start
  int *t_len, *t_lo, *d_len, *d_lo;
  int64_t *t_last, *d_last, *pending, *drafted, *accepted;
};

// the normalised fixed-point mass of a kept mass m out of a kept total M (Md = M rounded to fp64)
__device__ __forceinline__ uint64_t norm_mass(uint64_t m, double Md) { return m ? __double2ull_rn((double)m * kMassUnit / Md) : 0; }

__device__ __forceinline__ uint32_t philox_x0(uint64_t seed, int pos, uint32_t word1) {
  return philox4x32_10((uint32_t)seed, (uint32_t)(seed >> 32), make_uint4((uint32_t)pos, word1, 0u, 0u)).x;
}

// The filtered distribution of one logit row: threshold key, min-p bound, max logit and the kept total.
struct RowDist {
  uint32_t t_key;
  float thr;
  double lmax_d, Md;
  __device__ __forceinline__ uint64_t kept(uint32_t key, const double& inv_t) const {
    return key >= t_key && key_value(key) >= thr ? key_mass(key, lmax_d, inv_t) : 0;
  }
};

__global__ void __launch_bounds__(kSampThreads) spec_accept_kernel(const SpecParams sp) {
  __shared__ uint64_t s_w[kSampWarps];
  __shared__ uint64_t s_hc[256], s_hm[256], s_lc[256], s_lm[256];
  __shared__ int s_bin[2];
  __shared__ uint64_t s_above;
  __shared__ double s_need;
  __shared__ int64_t s_tok;

  const SampleParams &p = sp.tp, &q = sp.dp;
  const int b = blockIdx.x, tid = threadIdx.x, T = sp.k + 1, V = p.V;
  if (p.active[b] == 0) return;  // a finished row writes nothing
  const int L = sp.t_len[b] - T;  // the verify step has advanced the target by T
  const uint64_t seed = (uint64_t)p.seeds[b];
  const double inv_t = p.inv_t;
  uint32_t k[8], kq[8];

  // keep-set and kept total of one row
  auto dist = [&](const SampleParams& sprm, const uint16_t* row, uint64_t best) {
    RowDist r;
    const float lmax = key_value((uint32_t)(best >> 32));
    r.lmax_d = lmax;
    r.thr = lmax + sprm.minp_off;
    r.t_key = keep_threshold(sprm, row, r.lmax_d, inv_t, k, s_hc, s_hm, s_lc, s_lm, s_bin, s_above, s_need);
    uint64_t own = 0;
    for (int i0 = tid * 8; i0 < V; i0 += kTile) {
      const int n = load8(sprm, row, i0, k);
      for (int j = 0; j < n; ++j) own += r.kept(k[j], inv_t);
    }
    uint64_t M;
    block_incl_scan(own, s_w, M);
    r.Md = (double)M;
    return r;
  };

  int n = 0;
  int64_t y = -1;
  for (int i = 1; i <= T; ++i) {
    const bool bonus = i == T;
    const uint16_t* prow = p.logits + ((int64_t)b * T + i - 1) * p.ld;
    const uint64_t pbest = row_best(p, prow, s_w, k);
    const int64_t amax = (int64_t)(0xFFFFFFFFu - (uint32_t)pbest);
    const int64_t d = bonus ? -1 : sp.tokens[(int64_t)b * T + i];
    if (p.temperature == 0.f) {
      if (d == amax) {
        ++n;
        continue;
      }
      y = amax;
      break;
    }
    const RowDist P = dist(p, prow, pbest);
    const uint16_t* qrow = bonus ? nullptr : q.logits + ((int64_t)(i - 1) * sp.B + b) * q.ld;
    RowDist Q{};
    if (!bonus) {
      Q = dist(q, qrow, row_best(q, qrow, s_w, k));
      const uint64_t pd = norm_mass(P.kept(order_key(prow[d]), inv_t), P.Md);
      const uint64_t qd = norm_mass(Q.kept(order_key(qrow[d]), inv_t), Q.Md);
      // (2r + 1)·Q[d] < 2^25·P[d] in 128 bits
      const uint64_t a = 2ull * (philox_x0(seed, L + i, 1u) >> 8) + 1ull;
      const uint64_t lhs_hi = __umul64hi(a, qd), lhs_lo = a * qd, rhs_hi = pd >> 39, rhs_lo = pd << 25;
      if (lhs_hi < rhs_hi || (lhs_hi == rhs_hi && lhs_lo < rhs_lo)) {
        ++n;
        continue;
      }
    }
    // y from max(0, P - Q) (the bonus: from P); a residual of zero mass (P <= Q everywhere, by rounding) falls back to P
    bool use_q = !bonus;
    auto weight = [&](int i0, uint64_t (&m8)[8]) {
      const int nn = i0 < V ? load8(p, prow, i0, k) : 0;
      if (use_q && nn > 0) load8(q, qrow, i0, kq);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const uint64_t pj = j < nn ? norm_mass(P.kept(k[j], inv_t), P.Md) : 0;
        const uint64_t qj = use_q && j < nn ? norm_mass(Q.kept(kq[j], inv_t), Q.Md) : 0;
        m8[j] = pj > qj ? pj - qj : 0;
      }
    };
    uint64_t R = 0;
    for (int pass = 0; pass < 2 && R == 0; ++pass) {
      use_q = use_q && pass == 0;
      uint64_t own = 0, m8[8];
      for (int i0 = tid * 8; i0 < V; i0 += kTile) {
        weight(i0, m8);
#pragma unroll
        for (int j = 0; j < 8; ++j) own += m8[j];
      }
      block_incl_scan(own, s_w, R);
    }
    const int64_t tok = inverse_cdf(V, draw_target(philox_x0(seed, L + i, 2u), R), weight, s_w, &s_tok);
    y = tok >= 0 ? tok : amax;  // target < R, so the draw always lands
    break;
  }

  if (tid != 0) return;
  int no = p.n_out[b];
  bool live = true;
  for (int e = 0; e <= n && live; ++e) {
    const int64_t tok = e < n ? sp.tokens[(int64_t)b * T + 1 + e] : y;
    p.history[(int64_t)b * p.max_new + no] = tok;
    ++no;
    if (no >= p.max_new || p.prompt_len[b] + no >= p.max_seq_len || tok == p.eos) live = false;
  }
  p.n_out[b] = no;
  if (!live) p.active[b] = 0;
  sp.drafted[b] += sp.k;
  sp.accepted[b] += n;
  // both caches keep the accepted prefix: the last token in them is the one at index L + n, y is pending
  const int64_t last = sp.tokens[(int64_t)b * T + n];
  const int lo = sp.lo_q[(int64_t)b * T + n];
  sp.t_len[b] = sp.d_len[b] = L + n + 1;
  sp.t_lo[b] = sp.d_lo[b] = lo;
  sp.t_last[b] = sp.d_last[b] = last;
  sp.pending[b] = y;
}

inline bool aligned(const void* ptr, uintptr_t a) { return ((uintptr_t)ptr & (a - 1)) == 0; }

inline bool knobs_ok(float temperature, int top_k, float top_p, float min_p) {
  return temperature >= 0.f && isfinite(temperature) && top_k >= 0 && top_p > 0.f && top_p <= 1.f && min_p >= 0.f && min_p <= 1.f;
}

// the knobs and row layout of one logit matrix
SampleParams sample_params(const void* logits, int64_t ld, int V, float temperature, int top_k, float top_p, float min_p) {
  SampleParams p{};
  p.logits = (const uint16_t*)logits;
  p.ld = ld;
  p.V = V;
  p.top_k = top_k;
  p.temperature = temperature;
  p.inv_t = temperature > 0.f ? 1.0 / (double)temperature : 0.0;
  p.top_p = top_p;
  p.minp_off = min_p > 0.f ? (float)((double)temperature * log((double)min_p)) : -INFINITY;
  p.vec = aligned(logits, 16) && ld % 8 == 0;
  return p;
}

}  // namespace

// Return codes, checked before the first CUDA call: -1 a required pointer is null (logits, seeds, positions, out), or only some of
// the bookkeeping pointers are; -3 an impossible shape (B < 1, V < 1, V >= 2^23, ld < V); -4 a sampling parameter out of range
// (temperature < 0 or not finite, top_k < 0, top_p outside (0, 1], min_p outside [0, 1]); -5 max_new or max_seq_len < 1 with
// bookkeeping; -6 a misaligned pointer (2 bytes for the logits, 8 for int64, 4 for int32).
//
// logits: bf16 [B, V] with row stride ld (elements); seeds int64 [B] (the Philox key), positions int32 [B] (the counter), out int64
// [B]. Bookkeeping, all null or none: an inactive row (active[b] == 0) writes nothing; an active row writes its token to out[b] and
// history[b, n_out[b]] (int64 [B, max_new]), increments n_out[b] (int32), and clears active[b] (uint8) when n_out reaches max_new,
// when prompt_len[b] + n_out reaches max_seq_len, or when the token is eos (eos < 0: none).
PB_EXPORT int pb_sample_tokens(const void* logits, int64_t ld, int B, int V, float temperature, int top_k, float top_p, float min_p,
                               const int64_t* seeds, const int* positions, int64_t* out, int64_t* history, int* n_out,
                               unsigned char* active, const int* prompt_len, int max_new, int max_seq_len, int64_t eos,
                               cudaStream_t stream) {
  if (logits == nullptr || seeds == nullptr || positions == nullptr || out == nullptr) return -1;
  const int book = (history != nullptr) + (n_out != nullptr) + (active != nullptr) + (prompt_len != nullptr);
  if (book != 0 && book != 4) return -1;
  if (B < 1 || V < 1 || V >= (1 << 23) || ld < V) return -3;
  if (!knobs_ok(temperature, top_k, top_p, min_p)) return -4;
  if (book == 4 && (max_new < 1 || max_seq_len < 1)) return -5;
  if (!aligned(logits, 2) || !aligned(seeds, 8) || !aligned(out, 8) || !aligned(history, 8) || !aligned(positions, 4) ||
      !aligned(n_out, 4) || !aligned(prompt_len, 4))
    return -6;
  SampleParams p = sample_params(logits, ld, V, temperature, top_k, top_p, min_p);
  p.seeds = seeds;
  p.positions = positions;
  p.out = out;
  p.history = history;
  p.n_out = n_out;
  p.active = active;
  p.prompt_len = prompt_len;
  p.max_new = max_new;
  p.max_seq_len = max_seq_len;
  p.eos = eos;
  sample_tokens_kernel<<<B, kSampThreads, 0, stream>>>(p);
  PB_CHECK_LAUNCH();
  return 0;
}

// One round of speculative decoding per row, after the draft's k + 1 decode steps and the target's verify step (the contract is
// ops.spec_accept's). Return codes as pb_sample_tokens' (every pointer is required), plus -7 for k outside [1, 15].
//
// target: bf16 logits [B, k+1, V] (row stride ldt), draft: bf16 [k, B, V] (row stride ldd); seeds int64 [B]; tokens int64 [B, k+1]
// (x, d_1 .. d_k); lo_q int32 [B, k+1] (pb_verify_advance's). For every active row: emits d_1 .. d_n, y into history / n_out through
// the stop rules of pb_sample_tokens (clearing active), adds k to drafted and n to accepted (int64 [B]), and sets both caches'
// len = L + n + 1, lo = lo_q[b, n], last_tok = tokens[b, n] (L = the target's len - k - 1), and pending[b] = y.
PB_EXPORT int pb_spec_accept(const void* target, int64_t ldt, const void* draft, int64_t ldd, int B, int k, int V, float temperature,
                             int top_k, float top_p, float min_p, const int64_t* seeds, const int64_t* tokens, const int* lo_q,
                             int* t_len, int* t_lo, int64_t* t_last, int* d_len, int* d_lo, int64_t* d_last, int64_t* pending,
                             int64_t* history, int* n_out, unsigned char* active, const int* prompt_len, int max_new,
                             int max_seq_len, int64_t eos, int64_t* drafted, int64_t* accepted, cudaStream_t stream) {
  const void* req[] = {target, draft, seeds, tokens, lo_q, t_len, t_lo, t_last, d_len, d_lo, d_last, pending, history, n_out, active,
                       prompt_len, drafted, accepted};
  for (const void* r : req)
    if (r == nullptr) return -1;
  if (k < 1 || k > 15) return -7;
  if (B < 1 || V < 1 || V >= (1 << 23) || ldt < V || ldd < V) return -3;
  if (!knobs_ok(temperature, top_k, top_p, min_p)) return -4;
  if (max_new < 1 || max_seq_len < 1) return -5;
  const void* a8[] = {seeds, tokens, t_last, d_last, pending, history, drafted, accepted};
  const void* a4[] = {lo_q, t_len, t_lo, d_len, d_lo, n_out, prompt_len};
  if (!aligned(target, 2) || !aligned(draft, 2)) return -6;
  for (const void* r : a8)
    if (!aligned(r, 8)) return -6;
  for (const void* r : a4)
    if (!aligned(r, 4)) return -6;
  SpecParams sp{};
  sp.tp = sample_params(target, ldt, V, temperature, top_k, top_p, min_p);
  sp.dp = sample_params(draft, ldd, V, temperature, top_k, top_p, min_p);
  sp.tp.seeds = seeds;
  sp.tp.history = history;
  sp.tp.n_out = n_out;
  sp.tp.active = active;
  sp.tp.prompt_len = prompt_len;
  sp.tp.max_new = max_new;
  sp.tp.max_seq_len = max_seq_len;
  sp.tp.eos = eos;
  sp.k = k;
  sp.B = B;
  sp.tokens = tokens;
  sp.lo_q = lo_q;
  sp.t_len = t_len;
  sp.t_lo = t_lo;
  sp.t_last = t_last;
  sp.d_len = d_len;
  sp.d_lo = d_lo;
  sp.d_last = d_last;
  sp.pending = pending;
  sp.drafted = drafted;
  sp.accepted = accepted;
  spec_accept_kernel<<<B, kSampThreads, 0, stream>>>(sp);
  PB_CHECK_LAUNCH();
  return 0;
}
