// Backward of the fused HGT edge kernel (see edge.cu for the forward and the lane mapping).
//
// Forward per destination i and head h:  s_e = <q_i, k_e>,  p_e = exp(s_e - m_i) / (l_i + 1e-16),
//                                         agg_i = sum_e p_e v_e            (k_e / v_e include the RTE rows)
// Given dagg_i:   dv_e = p_e * dagg_i          dp_e = <dagg_i, v_e>          D_i = <dagg_i, agg_i> (= sum_e p_e dp_e)
//                 ds_e = p_e * (dp_e - D_i)    dq_i = sum_e ds_e k_e         dk_e = ds_e * q_i
// One pass over the destination-sorted CSR; p is recomputed from the saved per-(destination, head) (m, l).
// dq is owned by the destination's warp (atomics only for split hub pieces); dk / dv are scattered into the
// [K'|V'] gradient table (and the RTE gradient table) with vector fp32 reductions (red.global.add.v4.f32):
// many edges share a <source, relation> row.  The trailing all-zero row collects the gradient of edges that
// matched no triple and is discarded by the caller.
//
// Deterministic variant (hgt_edge_backward_dst + hgt_edge_backward_rows, chosen by the caller under
// torch.use_deterministic_algorithms): every gradient row has one owner and no float atomics are used.
//   destination pass  the same walk without the dk / dv scatter; writes dq (hub pieces: partial rows merged in piece
//                     order) and D_i = <dagg_i, agg_i> per head;
//   row pass          one warp owns a [K'|V'] row (or an RTE row) and walks its edges in a source-major index
//                     (hgt_plan_source_index): per edge it gathers Q_i, dagg_i, (m, l)_i, D_i and the other table's row,
//                     recomputes p / ds and accumulates dK = sum ds Q_i, dV = sum p dagg_i in registers; rows with more
//                     than the split threshold of edges are cut into pieces whose partial rows are merged in piece order.
//
// hgt_edge_backward*_bf16: the same passes on bf16 [K'|V'] / RTE tables (KV = __nv_bfloat16), widened to fp32 in registers;
// every gradient stays fp32 in the layouts above.
//
// Gradient of att as well (ATT = true, the *_att entry points): with an incoming datt_e (the loss reads att itself)
//                 C_i = sum_e p_e datt_e       ds_e = p_e * ((dp_e + datt_e) - (D_i + C_i))
// and dq / dk / dv as above.  hgt_edge_att_grad_prep computes C [N, H] and datt permuted to CSR order (one warp per
// destination tile, hub pieces merged in piece order: no float atomics, so it serves both backward modes); the passes
// read datt at the edge's CSR position (the row pass through a per-entry position beside its source-major index) and
// add C_i to D_i once per destination.  With datt = 0 the grouping gives bitwise the ds of the ATT = false passes.
#include <cuda_bf16.h>

#include "common.cuh"

#include <type_traits>

namespace {

constexpr int kWarps = 8;

struct BwdParams {
  const float* q;
  const void* kv;             // KV elements (float or bf16)
  const void* kvr;
  const float* agg;
  const float* dagg;
  const float* stats;        // [N, 2H] (m, l)
  const int32_t* row_ptr;
  const int32_t* kv_row;
  const int32_t* rte_row;
  const int32_t* tiles;
  int32_t n_tiles;
  const int32_t* d_counts;   // optional device {n_tiles, ...} (sync-free plans): n_tiles is then an upper bound
  int32_t d, H, DK, LPH, lph_shift;
  float* dq;                 // [N, d]   zero-initialised by hgt_edge_backward
  float* dkv;                // [rows+1, 2d] zero-initialised
  float* dkvr;               // [P*240+1, 2d] zero-initialised or nullptr
  int32_t* tile_counter;
  float* D;                  // deterministic destination pass: [N, H] D_i per head (+ C_i with ATT)
  float* partial;            // deterministic destination pass: [n_split, d] partial dq of hub pieces
  const float* datt_csr;     // ATT: [E, H] gradient of att in CSR order
  const float* c_att;        // ATT: [N, H] C_i = sum_e p_e datt_e
};

template <int VEC>
__device__ __forceinline__ void ld_vec(float (&dst)[VEC], const float* p) {
  if constexpr (VEC == 4) {
    float4 t = *reinterpret_cast<const float4*>(p);
    dst[0] = t.x; dst[1] = t.y; dst[2] = t.z; dst[3] = t.w;
  } else if constexpr (VEC == 2) {
    float2 t = *reinterpret_cast<const float2*>(p);
    dst[0] = t.x; dst[1] = t.y;
  } else {
    dst[0] = *p;
  }
}
template <int VEC>
__device__ __forceinline__ void ld_vec(float (&dst)[VEC], const __nv_bfloat16* p) {
  // bf16 -> fp32 is exact: the element is the high half of the fp32 word
  if constexpr (VEC == 4) {
    const uint2 u = *reinterpret_cast<const uint2*>(p);
    dst[0] = __uint_as_float(u.x << 16); dst[1] = __uint_as_float(u.x & 0xffff0000u);
    dst[2] = __uint_as_float(u.y << 16); dst[3] = __uint_as_float(u.y & 0xffff0000u);
  } else if constexpr (VEC == 2) {
    const uint32_t u = *reinterpret_cast<const uint32_t*>(p);
    dst[0] = __uint_as_float(u << 16); dst[1] = __uint_as_float(u & 0xffff0000u);
  } else {
    dst[0] = __bfloat162float(*p);
  }
}
template <int VEC>
__device__ __forceinline__ void red_add_vec(float* p, const float (&v)[VEC]) {
  if constexpr (VEC == 4) {
    asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v[0]), "f"(v[1]), "f"(v[2]), "f"(v[3])
                 : "memory");
  } else if constexpr (VEC == 2) {
    asm volatile("red.global.add.v2.f32 [%0], {%1,%2};" ::"l"(p), "f"(v[0]), "f"(v[1]) : "memory");
  } else {
    asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v[0]) : "memory");
  }
}
__device__ __forceinline__ float head_sum(float v, int lph) {
  for (int o = lph >> 1; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <int VEC>
__device__ __forceinline__ void st_vec(float* p, const float (&v)[VEC]) {
  if constexpr (VEC == 4) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  } else if constexpr (VEC == 2) {
    *reinterpret_cast<float2*>(p) = make_float2(v[0], v[1]);
  } else {
    *p = v[0];
  }
}

// DET = false: hgt_edge_backward (dk / dv scattered with reductions).  DET = true: destination pass of the
// deterministic backward (no scatter; D_i saved; hub pieces write partial dq rows).  ATT: datt_e and C_i enter ds.
template <class KV, int VEC, int NCH, bool DET, bool ATT>
__device__ __forceinline__ void edge_bwd_dst(const BwdParams& p) {
  const KV* const kvt = static_cast<const KV*>(p.kv);
  const KV* const kvrt = static_cast<const KV*>(p.kvr);
  const int lane = threadIdx.x & 31;
  const int lph = p.LPH;
  const int h = lane >> p.lph_shift;
  const int sub = lane & (lph - 1);
  const bool head_ok = h < p.H;
  int offs[NCH];
#pragma unroll
  for (int t = 0; t < NCH; ++t) {
    int o = (sub + t * lph) * VEC;
    offs[t] = (head_ok && o < p.DK) ? h * p.DK + o : -1;
  }
  const int64_t row_stride = 2 * (int64_t)p.d;
  const bool rte = kvrt != nullptr;

  const int n_tiles = p.d_counts ? p.d_counts[0] : p.n_tiles;
  for (;;) {
    int tile = 0;
    if (lane == 0) tile = atomicAdd(p.tile_counter, 1);
    tile = __shfl_sync(0xffffffffu, tile, 0);
    if (tile >= n_tiles) break;
    const int4 tl = reinterpret_cast<const int4*>(p.tiles)[tile];
    const bool split = tl.y < 0;
    const int d_begin = tl.x, d_end = split ? tl.x + 1 : tl.y;
    int seg_begin = tl.z;
    for (int dst = d_begin; dst < d_end; ++dst) {
      const int seg_end = split ? tl.w : p.row_ptr[dst + 1];
      if (seg_end > seg_begin) {
        float q[NCH][VEC], da[NCH][VEC], dq[NCH][VEC];
        float dpart = 0.f;
#pragma unroll
        for (int t = 0; t < NCH; ++t) {
          if (offs[t] >= 0) {
            float ag[VEC];
            ld_vec<VEC>(q[t], p.q + (int64_t)dst * p.d + offs[t]);
            ld_vec<VEC>(da[t], p.dagg + (int64_t)dst * p.d + offs[t]);
            ld_vec<VEC>(ag, p.agg + (int64_t)dst * p.d + offs[t]);
#pragma unroll
            for (int v = 0; v < VEC; ++v) dpart = fmaf(da[t][v], ag[v], dpart);
          } else {
#pragma unroll
            for (int v = 0; v < VEC; ++v) { q[t][v] = 0.f; da[t][v] = 0.f; }
          }
#pragma unroll
          for (int v = 0; v < VEC; ++v) dq[t][v] = 0.f;
        }
        const float D = ATT ? head_sum(dpart, lph) + (head_ok ? p.c_att[(int64_t)dst * p.H + h] : 0.f)
                            : head_sum(dpart, lph);
        if constexpr (DET) {
          if (head_ok && sub == 0 && seg_begin == p.row_ptr[dst]) p.D[(int64_t)dst * p.H + h] = D;
        }
        float m = 0.f, inv_l = 0.f;
        if (head_ok) {
          m = p.stats[(int64_t)dst * 2 * p.H + h];
          inv_l = 1.0f / (p.stats[(int64_t)dst * 2 * p.H + p.H + h] + 1e-16f);
        }
        for (int c = seg_begin; c < seg_end; ++c) {
          const int64_t row = p.kv_row[c];
          const int64_t rrow = rte ? p.rte_row[c] : 0;
          const KV* kvp = kvt + row * row_stride;
          float kk[NCH][VEC], vv[NCH][VEC];
          float spart = 0.f, dppart = 0.f;
#pragma unroll
          for (int t = 0; t < NCH; ++t) {
            if (offs[t] >= 0) {
              ld_vec<VEC>(kk[t], kvp + offs[t]);
              ld_vec<VEC>(vv[t], kvp + p.d + offs[t]);
              if (rte) {
                float a[VEC], b[VEC];
                ld_vec<VEC>(a, kvrt + rrow * row_stride + offs[t]);
                ld_vec<VEC>(b, kvrt + rrow * row_stride + p.d + offs[t]);
#pragma unroll
                for (int v = 0; v < VEC; ++v) { kk[t][v] += a[v]; vv[t][v] += b[v]; }
              }
#pragma unroll
              for (int v = 0; v < VEC; ++v) {
                spart = fmaf(q[t][v], kk[t][v], spart);
                dppart = fmaf(da[t][v], vv[t][v], dppart);
              }
            }
          }
          const float s = head_sum(spart, lph);
          const float dp = head_sum(dppart, lph);
          const float pe = __expf(s - m) * inv_l;
          float ds;
          if constexpr (ATT) {
            const float dat = head_ok ? p.datt_csr[(int64_t)c * p.H + h] : 0.f;
            ds = pe * ((dp + dat) - D);
          } else {
            ds = pe * (dp - D);
          }
          if constexpr (DET) {
#pragma unroll
            for (int t = 0; t < NCH; ++t)
              if (offs[t] >= 0) {
#pragma unroll
                for (int v = 0; v < VEC; ++v) dq[t][v] = fmaf(ds, kk[t][v], dq[t][v]);
              }
          } else {
            float* gk = p.dkv + row * row_stride;
#pragma unroll
            for (int t = 0; t < NCH; ++t) {
              if (offs[t] >= 0) {
                float gkv[VEC], gvv[VEC];
#pragma unroll
                for (int v = 0; v < VEC; ++v) {
                  dq[t][v] = fmaf(ds, kk[t][v], dq[t][v]);
                  gkv[v] = ds * q[t][v];
                  gvv[v] = pe * da[t][v];
                }
                red_add_vec<VEC>(gk + offs[t], gkv);
                red_add_vec<VEC>(gk + p.d + offs[t], gvv);
                if (rte) {
                  red_add_vec<VEC>(p.dkvr + rrow * row_stride + offs[t], gkv);
                  red_add_vec<VEC>(p.dkvr + rrow * row_stride + p.d + offs[t], gvv);
                }
              }
            }
          }
        }
        float* gq = p.dq + (int64_t)dst * p.d;
        if constexpr (DET) {
          if (split) gq = p.partial + (int64_t)(-tl.y - 1) * p.d;
#pragma unroll
          for (int t = 0; t < NCH; ++t)
            if (offs[t] >= 0) st_vec<VEC>(gq + offs[t], dq[t]);
        } else {
#pragma unroll
          for (int t = 0; t < NCH; ++t) {
            if (offs[t] >= 0) {
              if (split) red_add_vec<VEC>(gq + offs[t], dq[t]);
              else {
#pragma unroll
                for (int v = 0; v < VEC; ++v) gq[offs[t] + v] = dq[t][v];
              }
            }
          }
        }
      }
      seg_begin = seg_end;
    }
  }
}

template <class KV, int VEC, int NCH, bool ATT>
__global__ void __launch_bounds__(kWarps * 32)
k_edge_bwd(BwdParams p) {
  edge_bwd_dst<KV, VEC, NCH, false, ATT>(p);
}

template <class KV, int VEC, int NCH, bool ATT>
__global__ void __launch_bounds__(kWarps * 32)
k_edge_bwd_dst(BwdParams p) {
  edge_bwd_dst<KV, VEC, NCH, true, ATT>(p);
}

// ---- deterministic row pass --------------------------------------------------------------------------------------------
struct RowParams {
  const float* q;
  const float* dagg;
  const float* stats;        // [N, 2H] (m, l)
  const float* D;            // [N, H] from the destination pass
  const void* own;           // table of the owned rows [rows, 2d] ([K'|V'] or the RTE table), KV elements
  const void* oth;           // the other table added to every edge's key / value row, or nullptr
  const int32_t* ptr;        // [n_rows + 1] source-major index over the owned rows
  const int32_t* e_dst;      // per index entry: destination (rank order)
  const int32_t* e_oth;      // per index entry: row of the other table (unused without oth)
  const int32_t* tiles;
  int32_t n_tiles;
  const int32_t* d_counts;
  int32_t d, H, DK, LPH, lph_shift;
  float* grad;               // [rows, 2d] gradient of the owned table
  float* partial;            // [n_split, 2d] partial rows of split row pieces
  int32_t* tile_counter;
  const float* datt_csr;     // ATT: [E, H] gradient of att in CSR order
  const int32_t* e_pos;      // ATT: per index entry: its CSR position
};

// grad may be own itself (fp32 tables; the in-place contract of hgt_edge_backward_rows in hgt_b200.h): a row is read
// only by its owning warp, before that warp's one store of it, or by the pieces of a split row, which store to
// `partial`.  Neither pointer is __restrict__, so own stays on coherent loads (no ld.global.nc).

// ATT: D holds D_i + C_i (destination pass) and datt_e is read at the entry's CSR position.
template <class KV, int VEC, int NCH, bool ATT>
__global__ void __launch_bounds__(kWarps * 32)
k_edge_bwd_rows(RowParams p) {
  const KV* const own = static_cast<const KV*>(p.own);
  const KV* const oth = static_cast<const KV*>(p.oth);
  const int lane = threadIdx.x & 31;
  const int lph = p.LPH;
  const int h = lane >> p.lph_shift;
  const int sub = lane & (lph - 1);
  const bool head_ok = h < p.H;
  int offs[NCH];
#pragma unroll
  for (int t = 0; t < NCH; ++t) {
    int o = (sub + t * lph) * VEC;
    offs[t] = (head_ok && o < p.DK) ? h * p.DK + o : -1;
  }
  const int64_t row_stride = 2 * (int64_t)p.d;
  const bool two = oth != nullptr;

  const int n_tiles = p.d_counts ? p.d_counts[0] : p.n_tiles;
  for (;;) {
    int tile = 0;
    if (lane == 0) tile = atomicAdd(p.tile_counter, 1);
    tile = __shfl_sync(0xffffffffu, tile, 0);
    if (tile >= n_tiles) break;
    const int4 tl = reinterpret_cast<const int4*>(p.tiles)[tile];
    const bool split = tl.y < 0;
    const int r_begin = tl.x, r_end = split ? tl.x + 1 : tl.y;
    int seg_begin = tl.z;
    for (int row = r_begin; row < r_end; ++row) {
      const int seg_end = split ? tl.w : p.ptr[row + 1];
      float ko[NCH][VEC], vo[NCH][VEC], gk[NCH][VEC], gv[NCH][VEC];
#pragma unroll
      for (int t = 0; t < NCH; ++t)
#pragma unroll
        for (int v = 0; v < VEC; ++v) { ko[t][v] = vo[t][v] = gk[t][v] = gv[t][v] = 0.f; }
      if (seg_end > seg_begin) {
        const KV* orow = own + (int64_t)row * row_stride;
#pragma unroll
        for (int t = 0; t < NCH; ++t)
          if (offs[t] >= 0) {
            ld_vec<VEC>(ko[t], orow + offs[t]);
            ld_vec<VEC>(vo[t], orow + p.d + offs[t]);
          }
      }
      for (int j = seg_begin; j < seg_end; ++j) {
        const int64_t i = p.e_dst[j];
        const KV* xrow = two ? oth + (int64_t)p.e_oth[j] * row_stride : nullptr;
        float q[NCH][VEC], da[NCH][VEC];
        float spart = 0.f, dppart = 0.f;
#pragma unroll
        for (int t = 0; t < NCH; ++t) {
          if (offs[t] >= 0) {
            float kk[VEC], vv[VEC];
            ld_vec<VEC>(q[t], p.q + i * p.d + offs[t]);
            ld_vec<VEC>(da[t], p.dagg + i * p.d + offs[t]);
#pragma unroll
            for (int v = 0; v < VEC; ++v) { kk[v] = ko[t][v]; vv[v] = vo[t][v]; }
            if (two) {
              float a[VEC], b[VEC];
              ld_vec<VEC>(a, xrow + offs[t]);
              ld_vec<VEC>(b, xrow + p.d + offs[t]);
#pragma unroll
              for (int v = 0; v < VEC; ++v) { kk[v] += a[v]; vv[v] += b[v]; }
            }
#pragma unroll
            for (int v = 0; v < VEC; ++v) {
              spart = fmaf(q[t][v], kk[v], spart);
              dppart = fmaf(da[t][v], vv[v], dppart);
            }
          } else {
#pragma unroll
            for (int v = 0; v < VEC; ++v) { q[t][v] = 0.f; da[t][v] = 0.f; }
          }
        }
        const float s = head_sum(spart, lph);
        const float dp = head_sum(dppart, lph);
        float m = 0.f, inv_l = 0.f, D = 0.f;
        if (head_ok) {
          m = p.stats[i * 2 * p.H + h];
          inv_l = 1.0f / (p.stats[i * 2 * p.H + p.H + h] + 1e-16f);
          D = p.D[i * p.H + h];
        }
        const float pe = __expf(s - m) * inv_l;
        float ds;
        if constexpr (ATT) {
          const float dat = head_ok ? p.datt_csr[(int64_t)p.e_pos[j] * p.H + h] : 0.f;
          ds = pe * ((dp + dat) - D);
        } else {
          ds = pe * (dp - D);
        }
#pragma unroll
        for (int t = 0; t < NCH; ++t)
#pragma unroll
          for (int v = 0; v < VEC; ++v) {
            gk[t][v] = fmaf(ds, q[t][v], gk[t][v]);
            gv[t][v] = fmaf(pe, da[t][v], gv[t][v]);
          }
      }
      float* out = split ? p.partial + (int64_t)(-tl.y - 1) * row_stride : p.grad + (int64_t)row * row_stride;
#pragma unroll
      for (int t = 0; t < NCH; ++t)
        if (offs[t] >= 0) {
          st_vec<VEC>(out + offs[t], gk[t]);
          st_vec<VEC>(out + p.d + offs[t], gv[t]);
        }
      seg_begin = seg_end;
    }
  }
}

// Hub pieces of either pass: out[row] = sum of the pieces' partial rows, added in piece order.  One CTA per hub.
__global__ void __launch_bounds__(256)
k_merge_piece_rows(const int32_t* __restrict__ hubs, const int32_t* __restrict__ d_counts, int n_hubs_host,
                   const float* __restrict__ partial, int width, float* __restrict__ out) {
  const int n_hubs = d_counts ? d_counts[2] : n_hubs_host;
  for (int hb = blockIdx.x; hb < n_hubs; hb += gridDim.x) {
    const int row = hubs[4 * hb], slot0 = hubs[4 * hb + 1], pieces = hubs[4 * hb + 2];
    for (int c = threadIdx.x; c < width; c += blockDim.x) {
      float s = 0.f;
      for (int i = 0; i < pieces; ++i) s += partial[(int64_t)(slot0 + i) * width + c];
      out[(int64_t)row * width + c] = s;
    }
  }
}

// C_i and datt in CSR order for the ATT passes.  One warp per destination tile (the edge tiles of the plan), static
// tile order; HP = next_pow2(H) lanes cover the heads of one edge and 32 / HP edges are walked side by side, so each
// edge's H weights are read and written as one contiguous run.  The lanes of a head are summed with a fixed butterfly;
// hub pieces write partial C rows that k_merge_piece_rows adds in piece order.  No float atomics: deterministic.
__global__ void __launch_bounds__(kWarps * 32)
k_att_grad_prep(const float* __restrict__ att, const float* __restrict__ datt, const int32_t* __restrict__ csr_eid,
                const int32_t* __restrict__ row_ptr, const int32_t* __restrict__ tiles, int n_tiles_host,
                const int32_t* __restrict__ d_counts, int H, int hp_shift, float* __restrict__ c_att,
                float* __restrict__ datt_csr, float* __restrict__ partial) {
  const int lane = threadIdx.x & 31;
  const int HP = 1 << hp_shift;
  const int h = lane & (HP - 1);
  const int first = lane >> hp_shift;
  const int step = 32 >> hp_shift;
  const bool head_ok = h < H;
  const int n_tiles = d_counts ? d_counts[0] : n_tiles_host;
  for (int tile = blockIdx.x * kWarps + (threadIdx.x >> 5); tile < n_tiles; tile += gridDim.x * kWarps) {
    const int4 tl = reinterpret_cast<const int4*>(tiles)[tile];
    const bool split = tl.y < 0;
    const int d_begin = tl.x, d_end = split ? tl.x + 1 : tl.y;
    int seg_begin = tl.z;
    for (int dst = d_begin; dst < d_end; ++dst) {
      const int seg_end = split ? tl.w : row_ptr[dst + 1];
      float acc = 0.f;
      if (head_ok) {
        for (int c = seg_begin + first; c < seg_end; c += step) {
          const int64_t e = csr_eid[c];
          const float g = datt[e * H + h];
          datt_csr[(int64_t)c * H + h] = g;
          acc = fmaf(att[e * H + h], g, acc);
        }
      }
      for (int o = 16; o >= HP; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (head_ok && first == 0) (split ? partial + (int64_t)(-tl.y - 1) * H : c_att + (int64_t)dst * H)[h] = acc;
      seg_begin = seg_end;
    }
  }
}

template <class KV, typename Params, int VEC, bool ATT>
int dispatch(const Params& p, int nch, int grid, cudaStream_t st, bool det) {
  if constexpr (std::is_same<Params, RowParams>::value) {
    switch (nch) {
      case 1: k_edge_bwd_rows<KV, VEC, 1, ATT><<<grid, kWarps * 32, 0, st>>>(p); break;
      case 2: k_edge_bwd_rows<KV, VEC, 2, ATT><<<grid, kWarps * 32, 0, st>>>(p); break;
      case 4: k_edge_bwd_rows<KV, VEC, 4, ATT><<<grid, kWarps * 32, 0, st>>>(p); break;
      case 8: k_edge_bwd_rows<KV, VEC, 8, ATT><<<grid, kWarps * 32, 0, st>>>(p); break;
      default: hgt_set_error("hgt_edge_backward_rows: unsupported chunk count %d", nch); return 1;
    }
  } else if (det) {
    switch (nch) {
      case 1: k_edge_bwd_dst<KV, VEC, 1, ATT><<<grid, kWarps * 32, 0, st>>>(p); break;
      case 2: k_edge_bwd_dst<KV, VEC, 2, ATT><<<grid, kWarps * 32, 0, st>>>(p); break;
      case 4: k_edge_bwd_dst<KV, VEC, 4, ATT><<<grid, kWarps * 32, 0, st>>>(p); break;
      case 8: k_edge_bwd_dst<KV, VEC, 8, ATT><<<grid, kWarps * 32, 0, st>>>(p); break;
      default: hgt_set_error("hgt_edge_backward_dst: unsupported chunk count %d", nch); return 1;
    }
  } else {
    switch (nch) {
      case 1: k_edge_bwd<KV, VEC, 1, ATT><<<grid, kWarps * 32, 0, st>>>(p); break;
      case 2: k_edge_bwd<KV, VEC, 2, ATT><<<grid, kWarps * 32, 0, st>>>(p); break;
      case 4: k_edge_bwd<KV, VEC, 4, ATT><<<grid, kWarps * 32, 0, st>>>(p); break;
      case 8: k_edge_bwd<KV, VEC, 8, ATT><<<grid, kWarps * 32, 0, st>>>(p); break;
      default: hgt_set_error("hgt_edge_backward: unsupported chunk count %d", nch); return 1;
    }
  }
  HGT_LAUNCH_CHECK();
  return 0;
}

// Lane mapping shared by every pass: LPH lanes per head, VEC floats per load, NCH chunks per lane.
struct LaneMap {
  int DK, LPH, lph_shift, vec, nch;
};

int lane_map(int d, int n_heads, LaneMap& m, const char* who) {
  HGT_REQUIRE(n_heads >= 1 && n_heads <= 32 && d % n_heads == 0, "%s: bad d=%d / n_heads=%d", who, d, n_heads);
  m.DK = d / n_heads;
  int hp = 1;
  while (hp < n_heads) hp <<= 1;
  m.LPH = 32 / hp;
  int shift = 0;
  while ((1 << shift) < m.LPH) ++shift;
  m.lph_shift = shift;
  m.vec = 1;
  for (int v : {4, 2})
    if (m.DK % v == 0 && m.DK / v >= m.LPH) { m.vec = v; break; }
  int chunks = (m.DK + m.vec * m.LPH - 1) / (m.vec * m.LPH);
  m.nch = 1;
  while (m.nch < chunks) m.nch <<= 1;
  HGT_REQUIRE(m.nch <= 8, "%s: head width d_k=%d needs %d chunks per lane (max 8)", who, m.DK, chunks);
  return 0;
}

template <class KV, bool ATT, typename Params>
int launch_pass(const Params& p, const LaneMap& lm, int n_tiles, cudaStream_t st, bool det) {
  HGT_CHECK_CUDA(cudaMemsetAsync(p.tile_counter, 0, sizeof(int32_t), st));
  int grid = hgt_sm_count() * 4;
  int max_ctas = (n_tiles + kWarps - 1) / kWarps;
  if (grid > max_ctas) grid = max_ctas;
  if (lm.vec == 4) return dispatch<KV, Params, 4, ATT>(p, lm.nch, grid, st, det);
  if (lm.vec == 2) return dispatch<KV, Params, 2, ATT>(p, lm.nch, grid, st, det);
  return dispatch<KV, Params, 1, ATT>(p, lm.nch, grid, st, det);
}

// The passes' ATT = false instances when datt_csr is NULL (the calls without an att gradient), ATT = true otherwise.
template <class KV, typename Params>
int launch_pass_att(const Params& p, const LaneMap& lm, int n_tiles, cudaStream_t st, bool det) {
  return p.datt_csr ? launch_pass<KV, true>(p, lm, n_tiles, st, det) : launch_pass<KV, false>(p, lm, n_tiles, st, det);
}

int merge_pieces(const int32_t* hubs, int32_t n_hubs, const int32_t* d_counts, const float* partial, int width,
                 float* out, cudaStream_t st) {
  if (n_hubs <= 0) return 0;
  const int grid = n_hubs < 4 * hgt_sm_count() ? n_hubs : 4 * hgt_sm_count();
  k_merge_piece_rows<<<grid, 256, 0, st>>>(hubs, d_counts, n_hubs, partial, width, out);
  HGT_LAUNCH_CHECK();
  return 0;
}

template <class KV>
int edge_backward(const float* q, const KV* kv, const KV* kvr, const float* agg, const float* dagg, const float* stats,
                  const float* datt_csr, const float* c_att, const int32_t* row_ptr, const int32_t* kv_row,
                  const int32_t* rte_row, const int32_t* tiles, int32_t n_tiles, int64_t n_nodes, int32_t d,
                  int32_t n_heads, int64_t kv_rows_total, int64_t kvr_rows_total, float* dq, float* dkv, float* dkvr,
                  void* workspace, size_t workspace_bytes, const int32_t* d_tile_counts, cudaStream_t st) {
  HGT_REQUIRE(n_heads >= 1 && n_heads <= 32 && d % n_heads == 0, "hgt_edge_backward: bad d=%d / n_heads=%d", d, n_heads);
  HGT_REQUIRE((kvr != nullptr) == (rte_row != nullptr) && (kvr != nullptr) == (dkvr != nullptr),
              "hgt_edge_backward: kvr, rte_row and dkvr must go together");
  HGT_REQUIRE(workspace && workspace_bytes >= 256, "hgt_edge_backward: workspace too small");
  HGT_REQUIRE((datt_csr != nullptr) == (c_att != nullptr), "hgt_edge_backward_att: datt_csr and c_att must go together");
  // the kernel accumulates (dk / dv of a <source, relation> row come from many edges): this call owns the initialisation
  if (n_nodes > 0) HGT_CHECK_CUDA(cudaMemsetAsync(dq, 0, (size_t)n_nodes * d * sizeof(float), st));
  if (kv_rows_total > 0) HGT_CHECK_CUDA(cudaMemsetAsync(dkv, 0, (size_t)kv_rows_total * 2 * d * sizeof(float), st));
  if (dkvr && kvr_rows_total > 0)
    HGT_CHECK_CUDA(cudaMemsetAsync(dkvr, 0, (size_t)kvr_rows_total * 2 * d * sizeof(float), st));
  if (n_nodes == 0 || n_tiles == 0) return 0;
  BwdParams p;
  p.q = q; p.kv = kv; p.kvr = kvr; p.agg = agg; p.dagg = dagg; p.stats = stats; p.row_ptr = row_ptr;
  p.kv_row = kv_row; p.rte_row = rte_row; p.tiles = tiles; p.n_tiles = n_tiles; p.d_counts = d_tile_counts; p.d = d; p.H = n_heads;
  LaneMap lm;
  int rc = lane_map(d, n_heads, lm, "hgt_edge_backward");
  if (rc) return rc;
  p.DK = lm.DK; p.LPH = lm.LPH; p.lph_shift = lm.lph_shift;
  p.dq = dq; p.dkv = dkv; p.dkvr = dkvr;
  p.tile_counter = reinterpret_cast<int32_t*>(workspace);
  p.D = nullptr; p.partial = nullptr;
  p.datt_csr = datt_csr; p.c_att = c_att;
  return launch_pass_att<KV>(p, lm, n_tiles, st, false);
}

}  // namespace

extern "C" int hgt_edge_backward(const float* q, const float* kv, const float* kvr, const float* agg,
                                 const float* dagg, const float* stats, const int32_t* row_ptr,
                                 const int32_t* kv_row, const int32_t* rte_row, const int32_t* tiles, int32_t n_tiles,
                                 int64_t n_nodes, int32_t d, int32_t n_heads, int64_t kv_rows_total,
                                 int64_t kvr_rows_total, float* dq, float* dkv, float* dkvr,
                                 void* workspace, size_t workspace_bytes, const int32_t* d_tile_counts, void* stream_) {
  return edge_backward<float>(q, kv, kvr, agg, dagg, stats, nullptr, nullptr, row_ptr, kv_row, rte_row, tiles, n_tiles,
                              n_nodes, d, n_heads, kv_rows_total, kvr_rows_total, dq, dkv, dkvr, workspace,
                              workspace_bytes, d_tile_counts, (cudaStream_t)stream_);
}

extern "C" int hgt_edge_backward_bf16(const float* q, const void* kv, const void* kvr, const float* agg,
                                      const float* dagg, const float* stats, const int32_t* row_ptr,
                                      const int32_t* kv_row, const int32_t* rte_row, const int32_t* tiles,
                                      int32_t n_tiles, int64_t n_nodes, int32_t d, int32_t n_heads,
                                      int64_t kv_rows_total, int64_t kvr_rows_total, float* dq, float* dkv,
                                      float* dkvr, void* workspace, size_t workspace_bytes,
                                      const int32_t* d_tile_counts, void* stream_) {
  return edge_backward<__nv_bfloat16>(q, static_cast<const __nv_bfloat16*>(kv), static_cast<const __nv_bfloat16*>(kvr),
                                      agg, dagg, stats, nullptr, nullptr, row_ptr, kv_row, rte_row, tiles, n_tiles,
                                      n_nodes, d, n_heads, kv_rows_total, kvr_rows_total, dq, dkv, dkvr, workspace,
                                      workspace_bytes, d_tile_counts, (cudaStream_t)stream_);
}

extern "C" int hgt_edge_backward_det_workspace_bytes(int32_t n_split_dst, int32_t n_split_rows, int32_t d,
                                                     size_t* out_bytes) {
  HGT_REQUIRE(out_bytes && d > 0 && n_split_dst >= 0 && n_split_rows >= 0,
              "hgt_edge_backward_det_workspace_bytes: bad argument");
  const size_t a = (size_t)n_split_dst * d, b = (size_t)n_split_rows * 2 * d;
  *out_bytes = 256 + sizeof(float) * (a > b ? a : b);
  return 0;
}

namespace {

template <class KV>
int edge_backward_dst(const float* q, const KV* kv, const KV* kvr, const float* agg, const float* dagg,
                      const float* stats, const float* datt_csr, const float* c_att, const int32_t* row_ptr,
                      const int32_t* kv_row, const int32_t* rte_row, const int32_t* tiles, int32_t n_tiles,
                      int32_t n_split, const int32_t* hubs, int32_t n_hubs, int64_t n_nodes, int32_t d, int32_t n_heads,
                      float* dq, float* D, void* workspace, size_t workspace_bytes, const int32_t* d_tile_counts,
                      cudaStream_t st) {
  HGT_REQUIRE((kvr != nullptr) == (rte_row != nullptr), "hgt_edge_backward_dst: kvr and rte_row must go together");
  HGT_REQUIRE(dq && D, "hgt_edge_backward_dst: NULL output");
  HGT_REQUIRE((datt_csr != nullptr) == (c_att != nullptr),
              "hgt_edge_backward_dst_att: datt_csr and c_att must go together");
  size_t need = 0;
  hgt_edge_backward_det_workspace_bytes(n_split > 0 ? n_split : 0, 0, d, &need);
  HGT_REQUIRE(workspace && workspace_bytes >= need, "hgt_edge_backward_dst: workspace too small (%zu < %zu)",
              workspace_bytes, need);
  HGT_REQUIRE(n_split <= 0 || (hubs && n_hubs > 0), "hgt_edge_backward_dst: split tiles present but no hub list given");
  // destinations without in-edges keep a zero dq
  if (n_nodes > 0) HGT_CHECK_CUDA(cudaMemsetAsync(dq, 0, (size_t)n_nodes * d * sizeof(float), st));
  if (n_nodes == 0 || n_tiles == 0) return 0;
  LaneMap lm;
  int rc = lane_map(d, n_heads, lm, "hgt_edge_backward_dst");
  if (rc) return rc;
  BwdParams p;
  p.q = q; p.kv = kv; p.kvr = kvr; p.agg = agg; p.dagg = dagg; p.stats = stats; p.row_ptr = row_ptr;
  p.kv_row = kv_row; p.rte_row = rte_row; p.tiles = tiles; p.n_tiles = n_tiles; p.d_counts = d_tile_counts;
  p.d = d; p.H = n_heads; p.DK = lm.DK; p.LPH = lm.LPH; p.lph_shift = lm.lph_shift;
  p.dq = dq; p.dkv = nullptr; p.dkvr = nullptr;
  p.tile_counter = reinterpret_cast<int32_t*>(workspace);
  p.D = D;
  p.partial = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + 256);
  p.datt_csr = datt_csr; p.c_att = c_att;
  if ((rc = launch_pass_att<KV>(p, lm, n_tiles, st, true))) return rc;
  return n_split > 0 ? merge_pieces(hubs, n_hubs, d_tile_counts, p.partial, d, dq, st) : 0;
}

template <class KV>
int edge_backward_rows(const float* q, const float* dagg, const float* stats, const float* D, const float* datt_csr,
                       const KV* own, const KV* oth, const int32_t* src_ptr, const int32_t* src_dst,
                       const int32_t* src_oth, const int32_t* src_pos, int32_t n_rows, int64_t own_rows_total,
                       const int32_t* tiles, int32_t n_tiles, int32_t n_split, const int32_t* hubs, int32_t n_hubs,
                       int32_t d, int32_t n_heads, float* grad, void* workspace, size_t workspace_bytes,
                       const int32_t* d_tile_counts, cudaStream_t st) {
  HGT_REQUIRE(own && grad && (oth == nullptr || src_oth), "hgt_edge_backward_rows: NULL argument");
  HGT_REQUIRE((datt_csr != nullptr) == (src_pos != nullptr),
              "hgt_edge_backward_rows_att: datt_csr and src_pos must go together");
  HGT_REQUIRE(n_rows >= 0 && own_rows_total >= n_rows, "hgt_edge_backward_rows: n_rows=%d own_rows_total=%lld", n_rows,
              (long long)own_rows_total);
  size_t need = 0;
  hgt_edge_backward_det_workspace_bytes(0, n_split > 0 ? n_split : 0, d, &need);
  HGT_REQUIRE(workspace && workspace_bytes >= need, "hgt_edge_backward_rows: workspace too small (%zu < %zu)",
              workspace_bytes, need);
  HGT_REQUIRE(n_split <= 0 || (hubs && n_hubs > 0), "hgt_edge_backward_rows: split tiles present but no hub list given");
  // rows past n_rows (the trailing all-zero row that collects unmatched edges) get no work: their gradient is zero
  if (own_rows_total > n_rows)
    HGT_CHECK_CUDA(cudaMemsetAsync(grad + (int64_t)n_rows * 2 * d, 0, (size_t)(own_rows_total - n_rows) * 2 * d * sizeof(float),
                                   st));
  if (n_rows == 0 || n_tiles == 0) return 0;
  LaneMap lm;
  int rc = lane_map(d, n_heads, lm, "hgt_edge_backward_rows");
  if (rc) return rc;
  RowParams p;
  p.q = q; p.dagg = dagg; p.stats = stats; p.D = D; p.own = own; p.oth = oth; p.ptr = src_ptr; p.e_dst = src_dst;
  p.e_oth = src_oth; p.tiles = tiles; p.n_tiles = n_tiles; p.d_counts = d_tile_counts;
  p.d = d; p.H = n_heads; p.DK = lm.DK; p.LPH = lm.LPH; p.lph_shift = lm.lph_shift;
  p.grad = grad;
  p.tile_counter = reinterpret_cast<int32_t*>(workspace);
  p.partial = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + 256);
  p.datt_csr = datt_csr; p.e_pos = src_pos;
  if ((rc = launch_pass_att<KV>(p, lm, n_tiles, st, true))) return rc;
  return n_split > 0 ? merge_pieces(hubs, n_hubs, d_tile_counts, p.partial, 2 * d, grad, st) : 0;
}

}  // namespace

extern "C" int hgt_edge_backward_dst(const float* q, const float* kv, const float* kvr, const float* agg,
                                     const float* dagg, const float* stats, const int32_t* row_ptr,
                                     const int32_t* kv_row, const int32_t* rte_row, const int32_t* tiles,
                                     int32_t n_tiles, int32_t n_split, const int32_t* hubs, int32_t n_hubs,
                                     int64_t n_nodes, int32_t d, int32_t n_heads, float* dq, float* D,
                                     void* workspace, size_t workspace_bytes, const int32_t* d_tile_counts,
                                     void* stream_) {
  return edge_backward_dst<float>(q, kv, kvr, agg, dagg, stats, nullptr, nullptr, row_ptr, kv_row, rte_row, tiles,
                                  n_tiles, n_split, hubs, n_hubs, n_nodes, d, n_heads, dq, D, workspace,
                                  workspace_bytes, d_tile_counts, (cudaStream_t)stream_);
}

extern "C" int hgt_edge_backward_dst_bf16(const float* q, const void* kv, const void* kvr, const float* agg,
                                          const float* dagg, const float* stats, const int32_t* row_ptr,
                                          const int32_t* kv_row, const int32_t* rte_row, const int32_t* tiles,
                                          int32_t n_tiles, int32_t n_split, const int32_t* hubs, int32_t n_hubs,
                                          int64_t n_nodes, int32_t d, int32_t n_heads, float* dq, float* D,
                                          void* workspace, size_t workspace_bytes, const int32_t* d_tile_counts,
                                          void* stream_) {
  return edge_backward_dst<__nv_bfloat16>(q, static_cast<const __nv_bfloat16*>(kv),
                                          static_cast<const __nv_bfloat16*>(kvr), agg, dagg, stats, nullptr, nullptr,
                                          row_ptr, kv_row,
                                          rte_row, tiles, n_tiles, n_split, hubs, n_hubs, n_nodes, d, n_heads, dq, D,
                                          workspace, workspace_bytes, d_tile_counts, (cudaStream_t)stream_);
}

extern "C" int hgt_edge_backward_rows(const float* q, const float* dagg, const float* stats, const float* D,
                                      const float* own, const float* oth, const int32_t* src_ptr,
                                      const int32_t* src_dst, const int32_t* src_oth, int32_t n_rows,
                                      int64_t own_rows_total, const int32_t* tiles, int32_t n_tiles, int32_t n_split,
                                      const int32_t* hubs, int32_t n_hubs, int32_t d, int32_t n_heads, float* grad,
                                      void* workspace, size_t workspace_bytes, const int32_t* d_tile_counts,
                                      void* stream_) {
  return edge_backward_rows<float>(q, dagg, stats, D, nullptr, own, oth, src_ptr, src_dst, src_oth, nullptr, n_rows,
                                   own_rows_total, tiles, n_tiles, n_split, hubs, n_hubs, d, n_heads, grad, workspace,
                                   workspace_bytes, d_tile_counts, (cudaStream_t)stream_);
}

extern "C" int hgt_edge_backward_rows_bf16(const float* q, const float* dagg, const float* stats, const float* D,
                                           const void* own, const void* oth, const int32_t* src_ptr,
                                           const int32_t* src_dst, const int32_t* src_oth, int32_t n_rows,
                                           int64_t own_rows_total, const int32_t* tiles, int32_t n_tiles,
                                           int32_t n_split, const int32_t* hubs, int32_t n_hubs, int32_t d,
                                           int32_t n_heads, float* grad, void* workspace, size_t workspace_bytes,
                                           const int32_t* d_tile_counts, void* stream_) {
  return edge_backward_rows<__nv_bfloat16>(q, dagg, stats, D, nullptr, static_cast<const __nv_bfloat16*>(own),
                                           static_cast<const __nv_bfloat16*>(oth), src_ptr, src_dst, src_oth, nullptr,
                                           n_rows, own_rows_total, tiles, n_tiles, n_split, hubs, n_hubs, d, n_heads,
                                           grad, workspace, workspace_bytes, d_tile_counts, (cudaStream_t)stream_);
}

// ---- gradient of att -------------------------------------------------------------------------------------------------

extern "C" int hgt_edge_att_grad_workspace_bytes(int32_t n_split, int32_t n_heads, size_t* out_bytes) {
  HGT_REQUIRE(out_bytes && n_split >= 0 && n_heads >= 1 && n_heads <= 32,
              "hgt_edge_att_grad_workspace_bytes: bad argument");
  *out_bytes = 256 + sizeof(float) * (size_t)n_split * n_heads;
  return 0;
}

extern "C" int hgt_edge_att_grad_prep(const float* att, const float* datt, const int32_t* csr_eid,
                                      const int32_t* row_ptr, const int32_t* tiles, int32_t n_tiles, int32_t n_split,
                                      const int32_t* hubs, int32_t n_hubs, int64_t n_nodes, int32_t n_heads,
                                      float* c_att, float* datt_csr, void* workspace, size_t workspace_bytes,
                                      const int32_t* d_tile_counts, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  HGT_REQUIRE(n_heads >= 1 && n_heads <= 32, "hgt_edge_att_grad_prep: bad n_heads=%d", n_heads);
  HGT_REQUIRE(c_att && datt_csr && (n_tiles == 0 || (att && datt && csr_eid && row_ptr && tiles)),
              "hgt_edge_att_grad_prep: NULL argument");
  size_t need = 0;
  hgt_edge_att_grad_workspace_bytes(n_split > 0 ? n_split : 0, n_heads, &need);
  HGT_REQUIRE(workspace && workspace_bytes >= need, "hgt_edge_att_grad_prep: workspace too small (%zu < %zu)",
              workspace_bytes, need);
  HGT_REQUIRE(n_split <= 0 || (hubs && n_hubs > 0), "hgt_edge_att_grad_prep: split tiles present but no hub list given");
  if (n_nodes == 0 || n_tiles == 0) return 0;
  int hp_shift = 0;
  while ((1 << hp_shift) < n_heads) ++hp_shift;
  int grid = hgt_sm_count() * 4;
  const int max_ctas = (n_tiles + kWarps - 1) / kWarps;
  if (grid > max_ctas) grid = max_ctas;
  float* partial = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + 256);
  k_att_grad_prep<<<grid, kWarps * 32, 0, st>>>(att, datt, csr_eid, row_ptr, tiles, n_tiles, d_tile_counts, n_heads,
                                                hp_shift, c_att, datt_csr, partial);
  HGT_LAUNCH_CHECK();
  return n_split > 0 ? merge_pieces(hubs, n_hubs, d_tile_counts, partial, n_heads, c_att, st) : 0;
}

extern "C" int hgt_edge_backward_att(const float* q, const float* kv, const float* kvr, const float* agg,
                                     const float* dagg, const float* stats, const float* datt_csr, const float* c_att,
                                     const int32_t* row_ptr, const int32_t* kv_row, const int32_t* rte_row,
                                     const int32_t* tiles, int32_t n_tiles, int64_t n_nodes, int32_t d, int32_t n_heads,
                                     int64_t kv_rows_total, int64_t kvr_rows_total, float* dq, float* dkv, float* dkvr,
                                     void* workspace, size_t workspace_bytes, const int32_t* d_tile_counts,
                                     void* stream_) {
  HGT_REQUIRE(datt_csr && c_att, "hgt_edge_backward_att: NULL datt_csr / c_att");
  return edge_backward<float>(q, kv, kvr, agg, dagg, stats, datt_csr, c_att, row_ptr, kv_row, rte_row, tiles, n_tiles,
                              n_nodes, d, n_heads, kv_rows_total, kvr_rows_total, dq, dkv, dkvr, workspace,
                              workspace_bytes, d_tile_counts, (cudaStream_t)stream_);
}

extern "C" int hgt_edge_backward_att_bf16(const float* q, const void* kv, const void* kvr, const float* agg,
                                          const float* dagg, const float* stats, const float* datt_csr,
                                          const float* c_att, const int32_t* row_ptr, const int32_t* kv_row,
                                          const int32_t* rte_row, const int32_t* tiles, int32_t n_tiles,
                                          int64_t n_nodes, int32_t d, int32_t n_heads, int64_t kv_rows_total,
                                          int64_t kvr_rows_total, float* dq, float* dkv, float* dkvr, void* workspace,
                                          size_t workspace_bytes, const int32_t* d_tile_counts, void* stream_) {
  HGT_REQUIRE(datt_csr && c_att, "hgt_edge_backward_att_bf16: NULL datt_csr / c_att");
  return edge_backward<__nv_bfloat16>(q, static_cast<const __nv_bfloat16*>(kv), static_cast<const __nv_bfloat16*>(kvr),
                                      agg, dagg, stats, datt_csr, c_att, row_ptr, kv_row, rte_row, tiles, n_tiles,
                                      n_nodes, d, n_heads, kv_rows_total, kvr_rows_total, dq, dkv, dkvr, workspace,
                                      workspace_bytes, d_tile_counts, (cudaStream_t)stream_);
}

extern "C" int hgt_edge_backward_dst_att(const float* q, const float* kv, const float* kvr, const float* agg,
                                         const float* dagg, const float* stats, const float* datt_csr,
                                         const float* c_att, const int32_t* row_ptr, const int32_t* kv_row,
                                         const int32_t* rte_row, const int32_t* tiles, int32_t n_tiles,
                                         int32_t n_split, const int32_t* hubs, int32_t n_hubs, int64_t n_nodes,
                                         int32_t d, int32_t n_heads, float* dq, float* D, void* workspace,
                                         size_t workspace_bytes, const int32_t* d_tile_counts, void* stream_) {
  HGT_REQUIRE(datt_csr && c_att, "hgt_edge_backward_dst_att: NULL datt_csr / c_att");
  return edge_backward_dst<float>(q, kv, kvr, agg, dagg, stats, datt_csr, c_att, row_ptr, kv_row, rte_row, tiles,
                                  n_tiles, n_split, hubs, n_hubs, n_nodes, d, n_heads, dq, D, workspace,
                                  workspace_bytes, d_tile_counts, (cudaStream_t)stream_);
}

extern "C" int hgt_edge_backward_dst_att_bf16(const float* q, const void* kv, const void* kvr, const float* agg,
                                              const float* dagg, const float* stats, const float* datt_csr,
                                              const float* c_att, const int32_t* row_ptr, const int32_t* kv_row,
                                              const int32_t* rte_row, const int32_t* tiles, int32_t n_tiles,
                                              int32_t n_split, const int32_t* hubs, int32_t n_hubs, int64_t n_nodes,
                                              int32_t d, int32_t n_heads, float* dq, float* D, void* workspace,
                                              size_t workspace_bytes, const int32_t* d_tile_counts, void* stream_) {
  HGT_REQUIRE(datt_csr && c_att, "hgt_edge_backward_dst_att_bf16: NULL datt_csr / c_att");
  return edge_backward_dst<__nv_bfloat16>(q, static_cast<const __nv_bfloat16*>(kv),
                                          static_cast<const __nv_bfloat16*>(kvr), agg, dagg, stats, datt_csr, c_att,
                                          row_ptr, kv_row, rte_row, tiles, n_tiles, n_split, hubs, n_hubs, n_nodes, d,
                                          n_heads, dq, D, workspace, workspace_bytes, d_tile_counts,
                                          (cudaStream_t)stream_);
}

extern "C" int hgt_edge_backward_rows_att(const float* q, const float* dagg, const float* stats, const float* D,
                                          const float* datt_csr, const float* own, const float* oth,
                                          const int32_t* src_ptr, const int32_t* src_dst, const int32_t* src_oth,
                                          const int32_t* src_pos, int32_t n_rows, int64_t own_rows_total,
                                          const int32_t* tiles, int32_t n_tiles, int32_t n_split, const int32_t* hubs,
                                          int32_t n_hubs, int32_t d, int32_t n_heads, float* grad, void* workspace,
                                          size_t workspace_bytes, const int32_t* d_tile_counts, void* stream_) {
  HGT_REQUIRE(datt_csr && src_pos, "hgt_edge_backward_rows_att: NULL datt_csr / src_pos");
  return edge_backward_rows<float>(q, dagg, stats, D, datt_csr, own, oth, src_ptr, src_dst, src_oth, src_pos, n_rows,
                                   own_rows_total, tiles, n_tiles, n_split, hubs, n_hubs, d, n_heads, grad, workspace,
                                   workspace_bytes, d_tile_counts, (cudaStream_t)stream_);
}

extern "C" int hgt_edge_backward_rows_att_bf16(const float* q, const float* dagg, const float* stats, const float* D,
                                               const float* datt_csr, const void* own, const void* oth,
                                               const int32_t* src_ptr, const int32_t* src_dst, const int32_t* src_oth,
                                               const int32_t* src_pos, int32_t n_rows, int64_t own_rows_total,
                                               const int32_t* tiles, int32_t n_tiles, int32_t n_split,
                                               const int32_t* hubs, int32_t n_hubs, int32_t d, int32_t n_heads,
                                               float* grad, void* workspace, size_t workspace_bytes,
                                               const int32_t* d_tile_counts, void* stream_) {
  HGT_REQUIRE(datt_csr && src_pos, "hgt_edge_backward_rows_att_bf16: NULL datt_csr / src_pos");
  return edge_backward_rows<__nv_bfloat16>(q, dagg, stats, D, datt_csr, static_cast<const __nv_bfloat16*>(own),
                                           static_cast<const __nv_bfloat16*>(oth), src_ptr, src_dst, src_oth, src_pos,
                                           n_rows, own_rows_total, tiles, n_tiles, n_split, hubs, n_hubs, d, n_heads,
                                           grad, workspace, workspace_bytes, d_tile_counts, (cudaStream_t)stream_);
}
