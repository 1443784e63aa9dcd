// Backward of the small stages around the typed GEMMs (training path; the reference differentiates the same ops with
// autograd, OAG/train_paper_field.py:249):
//   hgt_update_backward   gated skip + LayerNorm (conv.py:129-133)  -> d o, d x, d skip, d norm.{weight,bias}
//   hgt_fold_backward     relation fold into the typed K/V weights (conv.py:97-99,103-104; hgt_fold_weights)
//                         -> d k_linears / v_linears (weight, bias), d relation_att / relation_msg / relation_pri
// The *_det entry points compute the same gradients without float atomics (torch.use_deterministic_algorithms): every
// output element has one owner, and partial sums are added in a fixed order.
// The DROP instances (hgt_update_backward_drop[_det]) take the PRE-dropout `o` and the forward's seed: they regenerate the
// mask (hgt_b200.h, "Fused dropout"), use o * mask * s wherever the others use o, and store d o * mask * s.
#include "common.cuh"

namespace {

// One warp per node row, ROWS_PER_WARP consecutive rows per warp; lane owns columns lane, lane+32, ...
// Forward:  y = o*a + x*(1-a),  a = sigmoid(skip[t]);   out = LayerNorm_t(y) = (y-mean)*rstd*w + b   (iff use_norm)
// Backward: dyh = dout*w;  dy = rstd*(dyh - mean(dyh) - yh*mean(dyh*yh));  do = a*dy;  dx = (1-a)*dy;
//           d a = sum dy*(o-x);  d skip[t] += d a * a*(1-a);  d w += dout*yh;  d b += dout.
constexpr int UB_WARPS = 8;
constexpr int UB_ROWS_PER_WARP = 16;

template <int NPL, bool DROP>
__global__ void __launch_bounds__(UB_WARPS * 32)
k_update_bwd(const float* __restrict__ dout, const float* __restrict__ o, const float* __restrict__ x,
             const int32_t* __restrict__ type_row0, int T, const float* __restrict__ skip,
             const float* __restrict__ norm_w, const int32_t* __restrict__ perm,
             const int32_t* __restrict__ type_active, int64_t n_nodes, int d,
             float* __restrict__ d_o, float* __restrict__ d_x, float* __restrict__ d_skip, float* __restrict__ d_nw,
             float* __restrict__ d_nb, const uint64_t* __restrict__ seed, uint32_t thr, float scale) {
  extern __shared__ float s_red[];                  // [2*d + 1] block-level partial sums (uniform-type blocks)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t block_row0 = (int64_t)blockIdx.x * UB_WARPS * UB_ROWS_PER_WARP;
  const int64_t block_row1 = min(n_nodes, block_row0 + UB_WARPS * UB_ROWS_PER_WARP);
  auto type_of = [&](int64_t row) {
    int t = 0;
    while (t < T && row >= type_row0[t + 1]) ++t;
    return t;
  };
  const int t_first = type_of(block_row0), t_last = type_of(block_row1 - 1);
  const bool uniform = t_first == t_last;
  for (int i = threadIdx.x; i < 2 * d + 1; i += blockDim.x) s_red[i] = 0.f;
  __syncthreads();

  float acc_w[NPL], acc_b[NPL];
  float acc_a = 0.f;
#pragma unroll
  for (int i = 0; i < NPL; ++i) acc_w[i] = acc_b[i] = 0.f;
  int cur_t = -1;
  auto flush = [&](int t) {
    if (t < 0 || t >= T) return;
    float da = 0.f;
    if (skip) {
      const float a = 1.0f / (1.0f + __expf(-skip[t]));
      da = acc_a;
      for (int s = 16; s > 0; s >>= 1) da += __shfl_xor_sync(0xffffffffu, da, s);
      da *= a * (1.0f - a);
    }
    if (uniform) {
      if (lane == 0 && skip) atomicAdd(&s_red[2 * d], da);
      if (norm_w) {
#pragma unroll
        for (int i = 0; i < NPL; ++i) {
          const int c = lane + 32 * i;
          if (c < d) { atomicAdd(&s_red[c], acc_w[i]); atomicAdd(&s_red[d + c], acc_b[i]); }
        }
      }
    } else {
      if (lane == 0 && skip) atomicAdd(d_skip + t, da);
      if (norm_w) {
#pragma unroll
        for (int i = 0; i < NPL; ++i) {
          const int c = lane + 32 * i;
          if (c < d) { atomicAdd(d_nw + (int64_t)t * d + c, acc_w[i]); atomicAdd(d_nb + (int64_t)t * d + c, acc_b[i]); }
        }
      }
    }
    acc_a = 0.f;
#pragma unroll
    for (int i = 0; i < NPL; ++i) acc_w[i] = acc_b[i] = 0.f;
  };

  const int64_t w_row0 = block_row0 + (int64_t)warp * UB_ROWS_PER_WARP;
  uint2 key = make_uint2(0u, 0u);
  if constexpr (DROP) key = hgt_drop_key(seed);
  for (int rr = 0; rr < UB_ROWS_PER_WARP; ++rr) {
    const int64_t row = w_row0 + rr;
    if (row >= n_nodes) break;
    const int t = type_of(row);
    if (t != cur_t) { flush(cur_t); cur_t = t; }
    float* dorow = d_o + row * d;
    float* dxrow = d_x + row * d;
    // unknown type: the forward wrote zeros (conv.py:120); rows past type_active[t] (sharded runs: halo sources) had no
    // output row at all: neither contributes a gradient, and their `o` rows were never computed
    if (t >= T || (type_active && row - type_row0[t] >= type_active[t])) {
#pragma unroll
      for (int i = 0; i < NPL; ++i) {
        const int c = lane + 32 * i;
        if (c < d) { dorow[c] = 0.f; dxrow[c] = 0.f; }
      }
      continue;
    }
    const float a = skip ? 1.0f / (1.0f + __expf(-skip[t])) : 1.0f;
    const float b1 = skip ? 1.0f - a : 1.0f;
    const float* gr = dout + (perm ? (int64_t)perm[row] : row) * d;
    const float* orow = o + row * d;
    const float* xrow = x + row * d;
    uint32_t kept = 0;
    if constexpr (DROP) kept = hgt_drop_row_bits<NPL>(key, row, d, thr, lane);
    float y[NPL], g[NPL], df[NPL];
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < NPL; ++i) {
      const int c = lane + 32 * i;
      if (c < d) {
        float ov = orow[c];
        const float xv = xrow[c];
        if constexpr (DROP) ov = hgt_drop_apply(ov, (kept >> i) & 1u, scale);
        g[i] = gr[c];
        df[i] = ov - xv;
        y[i] = ov * a + xv * b1;
        sum += y[i];
      } else {
        g[i] = df[i] = y[i] = 0.f;
      }
    }
    if (norm_w) {
      for (int s = 16; s > 0; s >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, s);
      const float mean = sum / d;
      float var = 0.f;
#pragma unroll
      for (int i = 0; i < NPL; ++i) {
        const int c = lane + 32 * i;
        if (c < d) { const float dl = y[i] - mean; var = fmaf(dl, dl, var); }
      }
      for (int s = 16; s > 0; s >>= 1) var += __shfl_xor_sync(0xffffffffu, var, s);
      const float rstd = rsqrtf(var / d + 1e-5f);
      const float* w = norm_w + (int64_t)t * d;
      float m1 = 0.f, m2 = 0.f;
#pragma unroll
      for (int i = 0; i < NPL; ++i) {
        const int c = lane + 32 * i;
        if (c < d) {
          const float yh = (y[i] - mean) * rstd;
          acc_w[i] = fmaf(g[i], yh, acc_w[i]);
          acc_b[i] += g[i];
          const float dyh = g[i] * w[c];
          y[i] = yh;
          g[i] = dyh;
          m1 += dyh;
          m2 = fmaf(dyh, yh, m2);
        }
      }
      for (int s = 16; s > 0; s >>= 1) {
        m1 += __shfl_xor_sync(0xffffffffu, m1, s);
        m2 += __shfl_xor_sync(0xffffffffu, m2, s);
      }
      m1 /= d;
      m2 /= d;
#pragma unroll
      for (int i = 0; i < NPL; ++i) g[i] = rstd * (g[i] - m1 - y[i] * m2);      // g := dy
    }
#pragma unroll
    for (int i = 0; i < NPL; ++i) {
      const int c = lane + 32 * i;
      if (c < d) {
        dorow[c] = DROP ? hgt_drop_apply(a * g[i], (kept >> i) & 1u, scale) : a * g[i];
        dxrow[c] = b1 * g[i];
        acc_a = fmaf(g[i], df[i], acc_a);
      }
    }
  }
  flush(cur_t);
  if (uniform) {
    __syncthreads();
    if (t_first < T) {
      if (norm_w) {
        for (int i = threadIdx.x; i < d; i += blockDim.x) {
          atomicAdd(d_nw + (int64_t)t_first * d + i, s_red[i]);
          atomicAdd(d_nb + (int64_t)t_first * d + i, s_red[d + i]);
        }
      }
      if (threadIdx.x == 0 && skip) atomicAdd(d_skip + t_first, s_red[2 * d]);
    }
  }
}

// ---- fold backward -----------------------------------------------------------------------------------------------------
// Forward (linear.cu k_fold_pairs):  W'[p,which][h*dk+c, col] = s * sum_a rel[r,h,a,c] * W[t][h*dk+a, col]  (col = d_in: bias)
// with rel = relation_att, s = pri[r,h]/sqrt(dk) for K' (which 0) and rel = relation_msg, s = 1 for V' (which 1).
// (a) d W[t][h*dk+a, col] += s * sum_c rel[a,c] * G[h*dk+c, col]           one thread per (p, which, row h*dk+a, col)
__global__ void k_fold_bwd_w(const float* __restrict__ g_w, const float* __restrict__ g_b,
                             const float* __restrict__ rel_att, const float* __restrict__ rel_msg,
                             const float* __restrict__ rel_pri, int H, int d_in, int d_out, int n_pairs,
                             const int32_t* __restrict__ pair_type, const int32_t* __restrict__ pair_rel,
                             const int32_t* __restrict__ cat_row0, float* __restrict__ d_wk, float* __restrict__ d_bk,
                             float* __restrict__ d_wv, float* __restrict__ d_bv) {
  const int dk = d_out / H;
  const int64_t per_block = (int64_t)d_out * (d_in + 1);
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= per_block * 2 * n_pairs) return;
  const int p = (int)(i / (2 * per_block));
  int64_t rem = i - (int64_t)p * 2 * per_block;
  const int which = (int)(rem / per_block);
  rem -= which * per_block;
  const int row = (int)(rem / (d_in + 1));
  const int col = (int)(rem - (int64_t)row * (d_in + 1));
  const int h = row / dk, a = row - h * dk;
  const int t = pair_type[p], r = pair_rel[p];
  const float* rel = (which ? rel_msg : rel_att) + ((int64_t)(r * H + h) * dk) * dk;   // [a][c]
  const int64_t g_row0 = (int64_t)cat_row0[p] + which * d_out + h * dk;
  float acc = 0.f;
  if (col < d_in) {
    for (int c = 0; c < dk; ++c) acc = fmaf(rel[a * dk + c], g_w[(g_row0 + c) * d_in + col], acc);
  } else {
    for (int c = 0; c < dk; ++c) acc = fmaf(rel[a * dk + c], g_b[g_row0 + c], acc);
  }
  if (!which) acc *= rel_pri[r * H + h] * rsqrtf((float)dk);
  if (col < d_in) atomicAdd((which ? d_wv : d_wk) + ((int64_t)t * d_out + row) * d_in + col, acc);
  else atomicAdd((which ? d_bv : d_bk) + (int64_t)t * d_out + row, acc);
}

// (b) val[a,c] = sum_col W[t][h*dk+a, col] * G[h*dk+c, col]  (bias column included);
//     d rel[r,h,a,c] += s * val;   d pri[r,h] += sum_{a,c} att[a,c] * val / sqrt(dk)   (K' only)
// One warp per (p, which, h, a, c); lanes split the columns.
__global__ void k_fold_bwd_rel(const float* __restrict__ g_w, const float* __restrict__ g_b,
                               const float* const* __restrict__ wk, const float* const* __restrict__ bk,
                               const float* const* __restrict__ wv, const float* const* __restrict__ bv,
                               const float* __restrict__ rel_att, const float* __restrict__ rel_pri, int H, int d_in,
                               int d_out, int n_pairs, const int32_t* __restrict__ pair_type,
                               const int32_t* __restrict__ pair_rel, const int32_t* __restrict__ cat_row0,
                               float* __restrict__ d_att, float* __restrict__ d_msg, float* __restrict__ d_pri) {
  const int dk = d_out / H;
  const int lane = threadIdx.x & 31;
  const int64_t wid = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t per_pair = (int64_t)2 * H * dk * dk;
  if (wid >= per_pair * n_pairs) return;
  const int p = (int)(wid / per_pair);
  int64_t rem = wid - (int64_t)p * per_pair;
  const int which = (int)(rem / ((int64_t)H * dk * dk));
  rem -= (int64_t)which * H * dk * dk;
  const int h = (int)(rem / (dk * dk));
  rem -= (int64_t)h * dk * dk;
  const int a = (int)(rem / dk), c = (int)(rem - (int64_t)a * dk);
  const int t = pair_type[p], r = pair_rel[p];
  const float* w = (which ? wv[t] : wk[t]) + (int64_t)(h * dk + a) * d_in;
  const int64_t g_row = (int64_t)cat_row0[p] + which * d_out + h * dk + c;
  const float* g = g_w + g_row * d_in;
  float val = 0.f;
  for (int col = lane; col < d_in; col += 32) val = fmaf(w[col], g[col], val);
  if (lane == 0) val = fmaf((which ? bv[t] : bk[t])[h * dk + a], g_b[g_row], val);
  for (int s = 16; s > 0; s >>= 1) val += __shfl_xor_sync(0xffffffffu, val, s);
  if (lane == 0) {
    const int64_t ridx = ((int64_t)(r * H + h) * dk + a) * dk + c;
    if (which) {
      atomicAdd(d_msg + ridx, val);
    } else {
      const float inv = rsqrtf((float)dk);
      atomicAdd(d_att + ridx, val * rel_pri[r * H + h] * inv);
      atomicAdd(d_pri + r * H + h, val * rel_att[ridx] * inv);
    }
  }
}

// ---- deterministic update backward ---------------------------------------------------------------------------------------
// Blocks never cross a type boundary: the blocks of type t are [blk0(t), blk0(t+1)) with ceil(count_t / UD_ROWS) blocks
// each (t = T: rows of unknown type, which only get zero gradients).  A block sums its rows' d norm / d skip terms warp by
// warp in warp order and stores them in its own partial slot [2d+1]; k_update_bwd_reduce adds a type's slots in block
// order.
constexpr int UD_ROWS_PER_WARP = 64;
constexpr int UD_ROWS = UB_WARPS * UD_ROWS_PER_WARP;

__device__ __forceinline__ int64_t ud_blocks_before(const int32_t* type_row0, int t) {
  int64_t b = 0;
  for (int u = 0; u < t; ++u) b += (type_row0[u + 1] - type_row0[u] + UD_ROWS - 1) / UD_ROWS;
  return b;
}

template <int NPL, bool DROP>
__global__ void __launch_bounds__(UB_WARPS * 32)
k_update_bwd_det(const float* __restrict__ dout, const float* __restrict__ o, const float* __restrict__ x,
                 const int32_t* __restrict__ type_row0, int T, const float* __restrict__ skip,
                 const float* __restrict__ norm_w, const int32_t* __restrict__ perm,
                 const int32_t* __restrict__ type_active, int d, float* __restrict__ d_o, float* __restrict__ d_x,
                 float* __restrict__ part, const uint64_t* __restrict__ seed, uint32_t thr, float scale) {
  extern __shared__ float s_red[];                  // [2*d + 1]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int t = 0;
  int64_t b0 = 0;
  for (; t <= T; ++t) {
    const int64_t nb = (type_row0[t + 1] - type_row0[t] + UD_ROWS - 1) / UD_ROWS;
    if (blockIdx.x < b0 + nb) break;
    b0 += nb;
  }
  if (t > T) return;                                 // grid is an upper bound
  const int64_t type_end = type_row0[t + 1];
  const int64_t block_row0 = type_row0[t] + (int64_t)(blockIdx.x - b0) * UD_ROWS;
  const bool known = t < T;
  const int64_t n_active = (known && type_active) ? (int64_t)type_row0[t] + type_active[t] : type_end;
  for (int i = threadIdx.x; i < 2 * d + 1; i += blockDim.x) s_red[i] = 0.f;

  float acc_w[NPL], acc_b[NPL];
  float acc_a = 0.f;
#pragma unroll
  for (int i = 0; i < NPL; ++i) acc_w[i] = acc_b[i] = 0.f;
  const float a = (known && skip) ? 1.0f / (1.0f + __expf(-skip[t])) : 1.0f;
  const float b1 = (known && skip) ? 1.0f - a : 1.0f;
  const int64_t w_row0 = block_row0 + (int64_t)warp * UD_ROWS_PER_WARP;
  uint2 key = make_uint2(0u, 0u);
  if constexpr (DROP) key = hgt_drop_key(seed);
  for (int rr = 0; rr < UD_ROWS_PER_WARP; ++rr) {
    const int64_t row = w_row0 + rr;
    if (row >= type_end) break;
    float* dorow = d_o + row * d;
    float* dxrow = d_x + row * d;
    if (!known || row >= n_active) {
#pragma unroll
      for (int i = 0; i < NPL; ++i) {
        const int c = lane + 32 * i;
        if (c < d) { dorow[c] = 0.f; dxrow[c] = 0.f; }
      }
      continue;
    }
    const float* gr = dout + (perm ? (int64_t)perm[row] : row) * d;
    const float* orow = o + row * d;
    const float* xrow = x + row * d;
    uint32_t kept = 0;
    if constexpr (DROP) kept = hgt_drop_row_bits<NPL>(key, row, d, thr, lane);
    float y[NPL], g[NPL], df[NPL];
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < NPL; ++i) {
      const int c = lane + 32 * i;
      if (c < d) {
        float ov = orow[c];
        const float xv = xrow[c];
        if constexpr (DROP) ov = hgt_drop_apply(ov, (kept >> i) & 1u, scale);
        g[i] = gr[c];
        df[i] = ov - xv;
        y[i] = ov * a + xv * b1;
        sum += y[i];
      } else {
        g[i] = df[i] = y[i] = 0.f;
      }
    }
    if (norm_w) {
      for (int s = 16; s > 0; s >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, s);
      const float mean = sum / d;
      float var = 0.f;
#pragma unroll
      for (int i = 0; i < NPL; ++i) {
        const int c = lane + 32 * i;
        if (c < d) { const float dl = y[i] - mean; var = fmaf(dl, dl, var); }
      }
      for (int s = 16; s > 0; s >>= 1) var += __shfl_xor_sync(0xffffffffu, var, s);
      const float rstd = rsqrtf(var / d + 1e-5f);
      const float* w = norm_w + (int64_t)t * d;
      float m1 = 0.f, m2 = 0.f;
#pragma unroll
      for (int i = 0; i < NPL; ++i) {
        const int c = lane + 32 * i;
        if (c < d) {
          const float yh = (y[i] - mean) * rstd;
          acc_w[i] = fmaf(g[i], yh, acc_w[i]);
          acc_b[i] += g[i];
          const float dyh = g[i] * w[c];
          y[i] = yh;
          g[i] = dyh;
          m1 += dyh;
          m2 = fmaf(dyh, yh, m2);
        }
      }
      for (int s = 16; s > 0; s >>= 1) {
        m1 += __shfl_xor_sync(0xffffffffu, m1, s);
        m2 += __shfl_xor_sync(0xffffffffu, m2, s);
      }
      m1 /= d;
      m2 /= d;
#pragma unroll
      for (int i = 0; i < NPL; ++i) g[i] = rstd * (g[i] - m1 - y[i] * m2);      // g := dy
    }
#pragma unroll
    for (int i = 0; i < NPL; ++i) {
      const int c = lane + 32 * i;
      if (c < d) {
        dorow[c] = DROP ? hgt_drop_apply(a * g[i], (kept >> i) & 1u, scale) : a * g[i];
        dxrow[c] = b1 * g[i];
        acc_a = fmaf(g[i], df[i], acc_a);
      }
    }
  }
  if (!known) return;                                // block-uniform: no partial slot for unknown rows
  for (int s = 16; s > 0; s >>= 1) acc_a += __shfl_xor_sync(0xffffffffu, acc_a, s);
  for (int w = 0; w < UB_WARPS; ++w) {               // warp order
    __syncthreads();
    if (warp == w) {
#pragma unroll
      for (int i = 0; i < NPL; ++i) {
        const int c = lane + 32 * i;
        if (c < d) { s_red[c] += acc_w[i]; s_red[d + c] += acc_b[i]; }
      }
      if (lane == 0) s_red[2 * d] += acc_a;
    }
  }
  __syncthreads();
  float* slot = part + (int64_t)blockIdx.x * (2 * d + 1);
  for (int i = threadIdx.x; i < 2 * d + 1; i += blockDim.x) slot[i] = s_red[i];
}

// One thread per (type, column of [d norm_w | d norm_b | d skip]): the type's block slots in block order.
__global__ void k_update_bwd_reduce(const float* __restrict__ part, const int32_t* __restrict__ type_row0, int T, int d,
                                    const float* __restrict__ skip, float* __restrict__ d_skip,
                                    float* __restrict__ d_nw, float* __restrict__ d_nb) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int w = 2 * d + 1;
  if (i >= (int64_t)T * w) return;
  const int t = (int)(i / w), c = (int)(i - (int64_t)t * w);
  if (c == 2 * d ? !d_skip : !d_nw) return;
  const int64_t b0 = ud_blocks_before(type_row0, t);
  const int64_t nb = (type_row0[t + 1] - type_row0[t] + UD_ROWS - 1) / UD_ROWS;
  float s = 0.f;
  for (int64_t b = 0; b < nb; ++b) s += part[(b0 + b) * w + c];
  if (c < d) d_nw[(int64_t)t * d + c] = s;
  else if (c < 2 * d) d_nb[(int64_t)t * d + c - d] = s;
  else {
    const float a = 1.0f / (1.0f + __expf(-skip[t]));
    d_skip[t] = s * a * (1.0f - a);
  }
}

// ---- deterministic fold backward ----------------------------------------------------------------------------------------
// (a) one thread per element of d W[t] / d b[t] (which, row, col): the pairs of source type t in pair order.
__global__ void k_fold_bwd_w_det(const float* __restrict__ g_w, const float* __restrict__ g_b,
                                 const float* __restrict__ rel_att, const float* __restrict__ rel_msg,
                                 const float* __restrict__ rel_pri, int T, int H, int d_in, int d_out, int n_pairs,
                                 const int32_t* __restrict__ pair_type, const int32_t* __restrict__ pair_rel,
                                 const int32_t* __restrict__ cat_row0, float* __restrict__ d_wk, float* __restrict__ d_bk,
                                 float* __restrict__ d_wv, float* __restrict__ d_bv) {
  const int dk = d_out / H;
  const int64_t per_block = (int64_t)d_out * (d_in + 1);
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= per_block * 2 * T) return;
  const int t = (int)(i / (2 * per_block));
  int64_t rem = i - (int64_t)t * 2 * per_block;
  const int which = (int)(rem / per_block);
  rem -= which * per_block;
  const int row = (int)(rem / (d_in + 1));
  const int col = (int)(rem - (int64_t)row * (d_in + 1));
  const int h = row / dk, a = row - h * dk;
  float sum = 0.f;
  for (int p = 0; p < n_pairs; ++p) {
    if (pair_type[p] != t) continue;
    const int r = pair_rel[p];
    const float* rel = (which ? rel_msg : rel_att) + ((int64_t)(r * H + h) * dk) * dk;
    const int64_t g_row0 = (int64_t)cat_row0[p] + which * d_out + h * dk;
    float acc = 0.f;
    if (col < d_in) {
      for (int c = 0; c < dk; ++c) acc = fmaf(rel[a * dk + c], g_w[(g_row0 + c) * d_in + col], acc);
    } else {
      for (int c = 0; c < dk; ++c) acc = fmaf(rel[a * dk + c], g_b[g_row0 + c], acc);
    }
    if (!which) acc *= rel_pri[r * H + h] * rsqrtf((float)dk);
    sum += acc;
  }
  if (col < d_in) (which ? d_wv : d_wk)[((int64_t)t * d_out + row) * d_in + col] = sum;
  else (which ? d_bv : d_bk)[(int64_t)t * d_out + row] = sum;
}

// (b) one warp per (r, which, h, a, c): V = sum over the pairs of relation r (pair order) of val; d_msg = V, and for K'
//     the raw V goes to d_att, scaled by k_fold_bwd_pri_det.
__global__ void k_fold_bwd_rel_det(const float* __restrict__ g_w, const float* __restrict__ g_b,
                                   const float* const* __restrict__ wk, const float* const* __restrict__ bk,
                                   const float* const* __restrict__ wv, const float* const* __restrict__ bv, int R, int H,
                                   int d_in, int d_out, int n_pairs, const int32_t* __restrict__ pair_type,
                                   const int32_t* __restrict__ pair_rel, const int32_t* __restrict__ cat_row0,
                                   float* __restrict__ d_att, float* __restrict__ d_msg) {
  const int dk = d_out / H;
  const int lane = threadIdx.x & 31;
  const int64_t wid = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t per_rel = (int64_t)2 * H * dk * dk;
  if (wid >= per_rel * R) return;
  const int r = (int)(wid / per_rel);
  int64_t rem = wid - (int64_t)r * per_rel;
  const int which = (int)(rem / ((int64_t)H * dk * dk));
  rem -= (int64_t)which * H * dk * dk;
  const int h = (int)(rem / (dk * dk));
  rem -= (int64_t)h * dk * dk;
  const int a = (int)(rem / dk), c = (int)(rem - (int64_t)a * dk);
  float sum = 0.f;
  for (int p = 0; p < n_pairs; ++p) {
    if (pair_rel[p] != r) continue;
    const int t = pair_type[p];
    const float* w = (which ? wv[t] : wk[t]) + (int64_t)(h * dk + a) * d_in;
    const int64_t g_row = (int64_t)cat_row0[p] + which * d_out + h * dk + c;
    const float* g = g_w + g_row * d_in;
    float val = 0.f;
    for (int col = lane; col < d_in; col += 32) val = fmaf(w[col], g[col], val);
    if (lane == 0) val = fmaf((which ? bv[t] : bk[t])[h * dk + a], g_b[g_row], val);
    for (int s = 16; s > 0; s >>= 1) val += __shfl_xor_sync(0xffffffffu, val, s);
    sum += val;
  }
  if (lane == 0) (which ? d_msg : d_att)[((int64_t)(r * H + h) * dk + a) * dk + c] = sum;
}

// (c) one warp per (r, h): d pri = sum_{a,c} att * V / sqrt(dk) (fixed lane split + butterfly), then d att = V * pri / sqrt(dk).
__global__ void k_fold_bwd_pri_det(const float* __restrict__ rel_att, const float* __restrict__ rel_pri, int R, int H,
                                   int dk, float* __restrict__ d_att, float* __restrict__ d_pri) {
  const int lane = threadIdx.x & 31;
  const int64_t wid = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  if (wid >= (int64_t)R * H) return;
  const float inv = rsqrtf((float)dk);
  const int64_t base = wid * dk * dk;
  const float pri = rel_pri[wid];
  float s = 0.f;
  for (int e = lane; e < dk * dk; e += 32) {
    const float v = d_att[base + e];
    s = fmaf(rel_att[base + e], v, s);
    d_att[base + e] = v * pri * inv;
  }
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) d_pri[wid] = s * inv;
}

template <int NPL, bool DROP>
void launch_update_bwd(const float* dout, const float* o, const float* x, const int32_t* type_row0, int T,
                       const float* skip, const float* norm_w, const int32_t* perm, const int32_t* type_active,
                       int64_t n, int d, float* d_o,
                       float* d_x, float* d_skip, float* d_nw, float* d_nb, const uint64_t* seed, HgtDrop dp,
                       cudaStream_t st) {
  const int rows_per_block = UB_WARPS * UB_ROWS_PER_WARP;
  const unsigned grid = (unsigned)((n + rows_per_block - 1) / rows_per_block);
  k_update_bwd<NPL, DROP><<<grid, UB_WARPS * 32, (2 * d + 1) * sizeof(float), st>>>(
      dout, o, x, type_row0, T, skip, norm_w, perm, type_active, n, d, d_o, d_x, d_skip, d_nw, d_nb, seed, dp.thr, dp.scale);
}

template <int NPL, bool DROP>
void launch_update_bwd_det(const float* dout, const float* o, const float* x, const int32_t* type_row0, int T,
                           const float* skip, const float* norm_w, const int32_t* perm, const int32_t* type_active,
                           unsigned grid, int d, float* d_o, float* d_x, float* part, const uint64_t* seed, HgtDrop dp,
                           cudaStream_t st) {
  k_update_bwd_det<NPL, DROP><<<grid, UB_WARPS * 32, (2 * d + 1) * sizeof(float), st>>>(
      dout, o, x, type_row0, T, skip, norm_w, perm, type_active, d, d_o, d_x, part, seed, dp.thr, dp.scale);
}

size_t update_det_slots(int64_t n_nodes, int32_t num_types) {
  return (size_t)((n_nodes + UD_ROWS - 1) / UD_ROWS + num_types + 1);
}

}  // namespace

static int update_backward_impl(const float* dout, const float* o, const float* x, const int32_t* type_row0,
                                int32_t num_types, const float* skip, const float* norm_w, const int32_t* perm,
                                const int32_t* type_active, int64_t n_nodes, int32_t d, float* d_o, float* d_x,
                                float* d_skip, float* d_norm_w, float* d_norm_b, const uint64_t* seed, float p,
                                cudaStream_t st) {
  HGT_REQUIRE(!seed || p > 0.f, "hgt_update_backward_drop: dropout needs p > 0");
  const HgtDrop dp = seed ? hgt_drop_params(p) : HgtDrop{0u, 1.f, 1.f};
  HGT_REQUIRE(dout && o && x && type_row0 && d_o && d_x && (d_skip || !skip), "hgt_update_backward: NULL argument");
  HGT_REQUIRE(d >= 1 && d <= 1024, "hgt_update_backward: d=%d unsupported (max 1024)", d);
  HGT_REQUIRE(!norm_w || (d_norm_w && d_norm_b), "hgt_update_backward: LayerNorm gradients need output buffers");
  if (skip) HGT_CHECK_CUDA(cudaMemsetAsync(d_skip, 0, (size_t)num_types * sizeof(float), st));
  if (norm_w) {
    HGT_CHECK_CUDA(cudaMemsetAsync(d_norm_w, 0, (size_t)num_types * d * sizeof(float), st));
    HGT_CHECK_CUDA(cudaMemsetAsync(d_norm_b, 0, (size_t)num_types * d * sizeof(float), st));
  }
  if (n_nodes == 0) return 0;
  const int npl = (d + 31) / 32;
#define HGT_UB(N)                                                                                                        \
  do {                                                                                                                   \
    if (seed) launch_update_bwd<N, true>(dout, o, x, type_row0, num_types, skip, norm_w, perm, type_active, n_nodes, d,   \
                                         d_o, d_x, d_skip, d_norm_w, d_norm_b, seed, dp, st);                            \
    else launch_update_bwd<N, false>(dout, o, x, type_row0, num_types, skip, norm_w, perm, type_active, n_nodes, d, d_o,  \
                                     d_x, d_skip, d_norm_w, d_norm_b, seed, dp, st);                                     \
  } while (0)
  if (npl <= 2) HGT_UB(2);
  else if (npl <= 4) HGT_UB(4);
  else if (npl <= 8) HGT_UB(8);
  else if (npl <= 16) HGT_UB(16);
  else HGT_UB(32);
#undef HGT_UB
  HGT_LAUNCH_CHECK();
  return 0;
}

extern "C" int hgt_update_backward(const float* dout, const float* o, const float* x, const int32_t* type_row0,
                                   int32_t num_types, const float* skip, const float* norm_w, const int32_t* perm,
                                   const int32_t* type_active, int64_t n_nodes, int32_t d, float* d_o, float* d_x, float* d_skip, float* d_norm_w,
                                   float* d_norm_b, void* stream_) {
  return update_backward_impl(dout, o, x, type_row0, num_types, skip, norm_w, perm, type_active, n_nodes, d, d_o, d_x,
                              d_skip, d_norm_w, d_norm_b, nullptr, 0.f, (cudaStream_t)stream_);
}

extern "C" int hgt_update_backward_drop(const float* dout, const float* o, const float* x, const int32_t* type_row0,
                                        int32_t num_types, const float* skip, const float* norm_w, const int32_t* perm,
                                        const int32_t* type_active, int64_t n_nodes, int32_t d, float* d_o, float* d_x,
                                        float* d_skip, float* d_norm_w, float* d_norm_b, const uint64_t* seed, float p,
                                        void* stream_) {
  HGT_REQUIRE(seed, "hgt_update_backward_drop: NULL seed");
  return update_backward_impl(dout, o, x, type_row0, num_types, skip, norm_w, perm, type_active, n_nodes, d, d_o, d_x,
                              d_skip, d_norm_w, d_norm_b, seed, p, (cudaStream_t)stream_);
}

extern "C" int hgt_fold_backward(const float* d_w_cat, const float* d_b_cat, const float* const* wk,
                                 const float* const* bk, const float* const* wv, const float* const* bv,
                                 const float* relation_att, const float* relation_msg, const float* relation_pri,
                                 int32_t num_types, int32_t num_relations, int32_t n_heads, int32_t d_in, int32_t d_out,
                                 int32_t n_pairs, const int32_t* pair_type, const int32_t* pair_rel,
                                 const int32_t* cat_row0, float* d_wk, float* d_bk, float* d_wv, float* d_bv,
                                 float* d_att, float* d_msg, float* d_pri, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  HGT_REQUIRE(n_heads > 0 && d_out % n_heads == 0, "hgt_fold_backward: d_out=%d not divisible by n_heads=%d", d_out, n_heads);
  HGT_REQUIRE(d_wk && d_bk && d_wv && d_bv && d_att && d_msg && d_pri, "hgt_fold_backward: NULL output");
  const int dk = d_out / n_heads;
  const size_t wbytes = (size_t)num_types * d_out * d_in * sizeof(float), bbytes = (size_t)num_types * d_out * sizeof(float);
  const size_t rbytes = (size_t)num_relations * n_heads * dk * dk * sizeof(float);
  HGT_CHECK_CUDA(cudaMemsetAsync(d_wk, 0, wbytes, st));
  HGT_CHECK_CUDA(cudaMemsetAsync(d_wv, 0, wbytes, st));
  HGT_CHECK_CUDA(cudaMemsetAsync(d_bk, 0, bbytes, st));
  HGT_CHECK_CUDA(cudaMemsetAsync(d_bv, 0, bbytes, st));
  HGT_CHECK_CUDA(cudaMemsetAsync(d_att, 0, rbytes, st));
  HGT_CHECK_CUDA(cudaMemsetAsync(d_msg, 0, rbytes, st));
  HGT_CHECK_CUDA(cudaMemsetAsync(d_pri, 0, (size_t)num_relations * n_heads * sizeof(float), st));
  if (n_pairs == 0) return 0;
  HGT_REQUIRE(d_w_cat && d_b_cat && wk && bk && wv && bv, "hgt_fold_backward: NULL input");
  {
    const int64_t total = (int64_t)n_pairs * 2 * d_out * (d_in + 1);
    k_fold_bwd_w<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(d_w_cat, d_b_cat, relation_att, relation_msg,
                                                                  relation_pri, n_heads, d_in, d_out, n_pairs, pair_type,
                                                                  pair_rel, cat_row0, d_wk, d_bk, d_wv, d_bv);
    HGT_LAUNCH_CHECK();
  }
  {
    const int64_t warps = (int64_t)n_pairs * 2 * n_heads * dk * dk;
    k_fold_bwd_rel<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, st>>>(d_w_cat, d_b_cat, wk, bk, wv, bv, relation_att,
                                                                        relation_pri, n_heads, d_in, d_out, n_pairs,
                                                                        pair_type, pair_rel, cat_row0, d_att, d_msg, d_pri);
    HGT_LAUNCH_CHECK();
  }
  return 0;
}

extern "C" int hgt_update_backward_det_workspace_bytes(int64_t n_nodes, int32_t num_types, int32_t d, size_t* out_bytes) {
  HGT_REQUIRE(out_bytes && n_nodes >= 0 && num_types >= 1 && d >= 1, "hgt_update_backward_det_workspace_bytes: bad argument");
  *out_bytes = update_det_slots(n_nodes, num_types) * (2 * (size_t)d + 1) * sizeof(float);
  return 0;
}

static int update_backward_det_impl(const float* dout, const float* o, const float* x, const int32_t* type_row0,
                                    int32_t num_types, const float* skip, const float* norm_w, const int32_t* perm,
                                    const int32_t* type_active, int64_t n_nodes, int32_t d, float* d_o, float* d_x,
                                    float* d_skip, float* d_norm_w, float* d_norm_b, void* workspace,
                                    size_t workspace_bytes, const uint64_t* seed, float p, cudaStream_t st) {
  HGT_REQUIRE(!seed || p > 0.f, "hgt_update_backward_drop_det: dropout needs p > 0");
  const HgtDrop dp = seed ? hgt_drop_params(p) : HgtDrop{0u, 1.f, 1.f};
  HGT_REQUIRE(dout && o && x && type_row0 && d_o && d_x && (d_skip || !skip), "hgt_update_backward_det: NULL argument");
  HGT_REQUIRE(d >= 1 && d <= 1024, "hgt_update_backward_det: d=%d unsupported (max 1024)", d);
  HGT_REQUIRE(!norm_w || (d_norm_w && d_norm_b), "hgt_update_backward_det: LayerNorm gradients need output buffers");
  size_t need = 0;
  hgt_update_backward_det_workspace_bytes(n_nodes, num_types, d, &need);
  HGT_REQUIRE(workspace && workspace_bytes >= need, "hgt_update_backward_det: workspace too small (%zu < %zu)",
              workspace_bytes, need);
  float* part = reinterpret_cast<float*>(workspace);
  if (n_nodes > 0) {
    const unsigned grid = (unsigned)update_det_slots(n_nodes, num_types);
    const int npl = (d + 31) / 32;
#define HGT_UBD(N)                                                                                                       \
  do {                                                                                                                   \
    if (seed) launch_update_bwd_det<N, true>(dout, o, x, type_row0, num_types, skip, norm_w, perm, type_active, grid, d,  \
                                             d_o, d_x, part, seed, dp, st);                                              \
    else launch_update_bwd_det<N, false>(dout, o, x, type_row0, num_types, skip, norm_w, perm, type_active, grid, d, d_o, \
                                         d_x, part, seed, dp, st);                                                       \
  } while (0)
    if (npl <= 2) HGT_UBD(2);
    else if (npl <= 4) HGT_UBD(4);
    else if (npl <= 8) HGT_UBD(8);
    else if (npl <= 16) HGT_UBD(16);
    else HGT_UBD(32);
#undef HGT_UBD
    HGT_LAUNCH_CHECK();
  }
  if (skip || norm_w) {
    const int64_t n = (int64_t)num_types * (2 * d + 1);
    k_update_bwd_reduce<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(part, type_row0, num_types, d, skip,
                                                                     skip ? d_skip : nullptr, norm_w ? d_norm_w : nullptr,
                                                                     d_norm_b);
    HGT_LAUNCH_CHECK();
  }
  return 0;
}

extern "C" int hgt_update_backward_det(const float* dout, const float* o, const float* x, const int32_t* type_row0,
                                       int32_t num_types, const float* skip, const float* norm_w, const int32_t* perm,
                                       const int32_t* type_active, int64_t n_nodes, int32_t d, float* d_o, float* d_x,
                                       float* d_skip, float* d_norm_w, float* d_norm_b, void* workspace,
                                       size_t workspace_bytes, void* stream_) {
  return update_backward_det_impl(dout, o, x, type_row0, num_types, skip, norm_w, perm, type_active, n_nodes, d, d_o, d_x,
                                  d_skip, d_norm_w, d_norm_b, workspace, workspace_bytes, nullptr, 0.f,
                                  (cudaStream_t)stream_);
}

extern "C" int hgt_update_backward_drop_det(const float* dout, const float* o, const float* x, const int32_t* type_row0,
                                            int32_t num_types, const float* skip, const float* norm_w,
                                            const int32_t* perm, const int32_t* type_active, int64_t n_nodes, int32_t d,
                                            float* d_o, float* d_x, float* d_skip, float* d_norm_w, float* d_norm_b,
                                            void* workspace, size_t workspace_bytes, const uint64_t* seed, float p,
                                            void* stream_) {
  HGT_REQUIRE(seed, "hgt_update_backward_drop_det: NULL seed");
  return update_backward_det_impl(dout, o, x, type_row0, num_types, skip, norm_w, perm, type_active, n_nodes, d, d_o, d_x,
                                  d_skip, d_norm_w, d_norm_b, workspace, workspace_bytes, seed, p, (cudaStream_t)stream_);
}

extern "C" int hgt_fold_backward_det(const float* d_w_cat, const float* d_b_cat, const float* const* wk,
                                     const float* const* bk, const float* const* wv, const float* const* bv,
                                     const float* relation_att, const float* relation_msg, const float* relation_pri,
                                     int32_t num_types, int32_t num_relations, int32_t n_heads, int32_t d_in, int32_t d_out,
                                     int32_t n_pairs, const int32_t* pair_type, const int32_t* pair_rel,
                                     const int32_t* cat_row0, float* d_wk, float* d_bk, float* d_wv, float* d_bv,
                                     float* d_att, float* d_msg, float* d_pri, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  HGT_REQUIRE(n_heads > 0 && d_out % n_heads == 0, "hgt_fold_backward_det: d_out=%d not divisible by n_heads=%d", d_out,
              n_heads);
  HGT_REQUIRE(d_wk && d_bk && d_wv && d_bv && d_att && d_msg && d_pri, "hgt_fold_backward_det: NULL output");
  HGT_REQUIRE(n_pairs == 0 || (d_w_cat && d_b_cat && wk && bk && wv && bv), "hgt_fold_backward_det: NULL input");
  const int dk = d_out / n_heads;
  // every output element is written (types / relations without pairs get zeros): no initialisation needed
  {
    const int64_t total = (int64_t)num_types * 2 * d_out * (d_in + 1);
    if (total > 0) {
      k_fold_bwd_w_det<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(d_w_cat, d_b_cat, relation_att, relation_msg,
                                                                        relation_pri, num_types, n_heads, d_in, d_out,
                                                                        n_pairs, pair_type, pair_rel, cat_row0, d_wk, d_bk,
                                                                        d_wv, d_bv);
      HGT_LAUNCH_CHECK();
    }
  }
  {
    const int64_t warps = (int64_t)num_relations * 2 * n_heads * dk * dk;
    if (warps > 0) {
      k_fold_bwd_rel_det<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, st>>>(d_w_cat, d_b_cat, wk, bk, wv, bv,
                                                                              num_relations, n_heads, d_in, d_out, n_pairs,
                                                                              pair_type, pair_rel, cat_row0, d_att, d_msg);
      HGT_LAUNCH_CHECK();
    }
  }
  {
    const int64_t warps = (int64_t)num_relations * n_heads;
    if (warps > 0) {
      k_fold_bwd_pri_det<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, st>>>(relation_att, relation_pri, num_relations,
                                                                              n_heads, dk, d_att, d_pri);
      HGT_LAUNCH_CHECK();
    }
  }
  return 0;
}
