// rb200_stream.cu — K1/K5/K6 for float-arithmetic op lists: the streaming kernel of the lean machine (sm_90a).
//
// What it stands for in the reference: the generated loop `for index in numba.pndindex(itershape): ...` over a
// contiguous 1-D (collapsed) iteration space (ramba/ramba.py:8246-8255), with the pre/postcode of a global reduction
// (`red[0] = red[0] + acc`, ramba/ramba.py:5798-5807), and the axis-reduction loop nest over a [rows][columns] box
// (ramba/ramba.py:8231-8244) - for op lists made of plain float arithmetic (rb200_plan.h).  Affine maps feeding
// a sum (`(X*2.0 + 1.0).sum()`), broadcast-add + column sums (`(M + v).sum(axis=0)`), float32 streams in general:
// at 4 bytes per element the general interpreter is bound by its own dispatch cost, this kernel by HBM.
//
//   * tile = 2048 consecutive elements (256 threads x 8, element k of thread t is k*256 + t: every access of a warp
//     is 32 consecutive elements);
//   * contiguous 16-byte aligned input views are STAGED: one elected thread issues one bulk async copy (TMA engine,
//     SASS UBLKCP) per view and tile into a ring of up to 8 stages, completion on an mbarrier - the ring holds the
//     bytes in flight that hide HBM latency, no registers are tied up by loads;
//   * mode 0 (elementwise / global reductions): persistent CTAs walk tiles b, b+grid, ...; reduction slots are
//     float64 accumulators in registers, folded warp -> CTA -> last CTA in a fixed order;
//   * mode 1 (axis reduction in column form): a CTA owns a chunk of 2048 columns and a slice of the rows, walks the
//     rows keeping 8 column accumulators per thread in registers, and writes partials[split][column]; operands that
//     are broadcast over the rows are loaded once into the shared-memory register file.
#include <cuda_runtime.h>
#include <stdio.h>
#include <string.h>

#include <string>

#include "rb200_launch.h"
#include "rb200_lean.cuh"
#include "rb200_plan.h"
#include "rb200_terms.h"
#include "rb200_mapred.h"
#include "rb200_stream.h"

namespace rb200 {

// element k of this thread in a staged tile of N * 256 elements of 4 (f32) or 8 bytes starting at `tile_s`
template <class F, int N> __device__ __forceinline__ void stream_lds(unsigned tile_s, unsigned tid, bool f32, F (&out)[N]) {
  if (f32) {
    const unsigned addr = tile_s + tid * 4u;
#pragma unroll
    for (int k = 0; k < N; ++k) out[k] = (F)lean_lds<float>(addr + k * kThreads * 4);
  } else {
    const unsigned addr = tile_s + tid * 8u;
#pragma unroll
    for (int k = 0; k < N; ++k) out[k] = (F)lean_lds<double>(addr + k * kThreads * 8);
  }
}

struct StreamCtx : LeanRegs {
  const StreamParams& P;
  unsigned stage_s;  // shared-window address of the current stage
  unsigned tid;
  bool staged_ok;    // the current tile was staged (false: ragged last tile, read directly)
  long long row, e0; // row (mode 1, else 0); element / column of k = 0
  unsigned valid;
  double racc[RB200_MAX_REDS];  // mode 0: reduction slots
  double cacc[LV];              // mode 1: column accumulators
  __device__ __forceinline__ StreamCtx(const StreamParams& p) : P(p) {}

  template <class F> __device__ __forceinline__ void fetch_direct(int arg, F (&out)[LV]) {
    const LDirect& v = P.direct[arg];
    ldirect_load<F, LV>(v, row * v.s1 + e0 * v.s2, (long long)kThreads * v.s2, valid, out);
  }
  template <class F> __device__ __forceinline__ void fetch(int kind, int arg, F (&out)[LV]) {
    switch (kind) {
      case L_STAGED: {
        const StreamStaged& sv = P.staged[arg];
        if (!staged_ok) {
          fetch_direct<F>(sv.dview, out);
          break;
        }
        stream_lds<F, LV>(stage_s + sv.off, tid, sv.es == 4, out);
      } break;
      case L_DIRECT: fetch_direct<F>(arg, out); break;
      case L_REG: fetch_reg<F>(arg, out); break;
      case L_SCAL: fetch_scal<F>(P.scal[arg], out); break;
      default: fetch_acc<F>(out);
    }
  }
  template <class F> __device__ __forceinline__ int chain_fetch(int, F (&)[LV]) { return 0; }  // (no chains in this kernel)
  template <class F> __device__ __forceinline__ void store_view(int arg, const F (&r)[LV]) {
    const LDirect& v = P.direct[arg];
    ldirect_store<F, LV>(v, row * v.s1 + e0 * v.s2, (long long)kThreads * v.s2, valid, r);
  }
  template <class F> __device__ __forceinline__ void reduce(int slot, int rop, const F (&a)[LV]) {
    if constexpr (sizeof(F) == 8) {
      if (P.mode == 1) {
#pragma unroll
        for (int k = 0; k < LV; ++k) cacc[k] = red_combine<double>(rop, cacc[k], a[k]);
        return;
      }
      double x[LV];
      const double ident = CT<double>::get(red_identity_bits(rop, RB200_T_F64));
#pragma unroll
      for (int k = 0; k < LV; ++k) x[k] = ((valid >> k) & 1u) ? (double)a[k] : ident;
#pragma unroll
      for (int w = LV / 2; w > 0; w >>= 1) {
#pragma unroll
        for (int k = 0; k < w; ++k) x[k] = red_combine<double>(rop, x[k], x[k + w]);
      }
#pragma unroll
      for (int s = 0; s < RB200_MAX_REDS; ++s)
        if (s == slot) racc[s] = red_combine<double>(rop, racc[s], x[0]);
    }
  }
};

// global reductions of a CTA's float64 accumulators: thread -> warp -> CTA -> per-CTA partial -> last CTA (fixed order,
// deterministic per grid); red[0,..] = red[0,..] (op) acc (ramba/ramba.py:5805-5806)
__device__ __forceinline__ void stream_finish_reductions(const StreamParams& P, const double (&racc)[RB200_MAX_REDS]) {
  // ---- global reductions: thread -> warp -> CTA -> per-CTA partial -> last CTA (fixed order, deterministic per grid)
  if (P.n_reds > 0) {
    __shared__ u64 wpart[RB200_MAX_REDS][kThreads / 32];
    __shared__ bool is_last;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int s = 0; s < P.n_reds; ++s) {
      const int op = P.reds[s].op;
      double mine = 0.0;
#pragma unroll
      for (int q = 0; q < RB200_MAX_REDS; ++q)
        if (q == s) mine = racc[q];
      u64 v = CT<double>::bits(mine);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v = red_combine_bits(op, RB200_T_F64, v, __shfl_down_sync(0xffffffffu, v, o));
      if (lane == 0) wpart[s][warp] = v;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int s = 0; s < P.n_reds; ++s) {
        const int op = P.reds[s].op;
        u64 v = wpart[s][0];
        for (int q = 1; q < kThreads / 32; ++q) v = red_combine_bits(op, RB200_T_F64, v, wpart[s][q]);
        P.red_partials[(long long)s * gridDim.x + blockIdx.x] = v;
      }
      __threadfence();
      const unsigned prev = atomicAdd(P.red_counter, 1u);
      is_last = (prev == gridDim.x - 1);
    }
    __syncthreads();
    if (is_last) {
      __threadfence();
      for (int s = 0; s < P.n_reds; ++s) {
        const int op = P.reds[s].op;
        u64 v = red_identity_bits(op, RB200_T_F64);
        for (unsigned b = threadIdx.x; b < gridDim.x; b += kThreads)
          v = red_combine_bits(op, RB200_T_F64, v, __ldcg(&P.red_partials[(long long)s * gridDim.x + b]));
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v = red_combine_bits(op, RB200_T_F64, v, __shfl_down_sync(0xffffffffu, v, o));
        __syncthreads();
        if (lane == 0) wpart[s][warp] = v;
        __syncthreads();
        if (threadIdx.x == 0) {
          v = wpart[s][0];
          for (int q = 1; q < kThreads / 32; ++q) v = red_combine_bits(op, RB200_T_F64, v, wpart[s][q]);
          // red[0,..] = red[0,..] (op) acc  (ramba/ramba.py:5805-5806), rounded to the partial array's dtype on store
          const double vd = CT<double>::get(v);
          void* out = P.reds[s].out;
          if (P.reds[s].out_dtype == RB200_F64) {
            double* o = (double*)out;
            *o = red_combine<double>(op, *o, vd);
          } else {
            float* o = (float*)out;
            *o = (float)red_combine<double>(op, (double)*o, vd);
          }
        }
      }
      if (threadIdx.x == 0) *P.red_counter = 0u;
    }
  }
}

__global__ void __launch_bounds__(kThreads, 2) stream_kernel(const __grid_constant__ StreamParams P) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const unsigned smem_s = (unsigned)__cvta_generic_to_shared(smem_raw);
  const unsigned tid = threadIdx.x;
  // layout: [ring: depth stages][register file: (n_regs + n_hoist) * 2048 * 8][mbarriers]
  const unsigned ring_bytes = (unsigned)P.depth * P.stage_bytes;
  const unsigned regs_s = smem_s + ring_bytes;
  const unsigned mbar_s = regs_s + (unsigned)(P.n_regs + P.n_hoist) * (LV * kThreads * 8);
  if (P.n_staged > 0 && tid == 0) {
    for (int s = 0; s < P.depth; ++s) mbar_init(mbar_s + 8u * s, 1u);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  StreamCtx cx(P);
  cx.tid = tid;
  cx.reg_s = regs_s + tid * 8u;
#pragma unroll
  for (int s = 0; s < RB200_MAX_REDS; ++s) cx.racc[s] = 0.0;
  for (int s = 0; s < P.n_reds; ++s) {
    const double ident = CT<double>::get(red_identity_bits(P.reds[s].op, RB200_T_F64));
#pragma unroll
    for (int q = 0; q < RB200_MAX_REDS; ++q)
      if (q == s) cx.racc[q] = ident;
  }

  // the CTA's sequence of tiles: it -> linear element offset of the tile inside the (contiguous) staged views
  long long n_it, base0, step_it;  // element offset of tile `it` = base0 + it * step_it
  long long split = 0, col0 = 0, r0 = 0;
  if (P.mode == 0) {
    n_it = (P.n_tiles - (long long)blockIdx.x + gridDim.x - 1) / gridDim.x;
    base0 = (long long)blockIdx.x * kStreamTile;
    step_it = (long long)gridDim.x * kStreamTile;
    cx.row = 0;
  } else {
    split = blockIdx.x / (unsigned)P.n_chunks;
    const long long chunk = blockIdx.x - split * P.n_chunks;
    col0 = chunk * kStreamTile;
    r0 = split * P.rows_per_split;
    long long r1 = r0 + P.rows_per_split;
    if (r1 > P.R) r1 = P.R;
    n_it = r1 > r0 ? r1 - r0 : 0;
    base0 = r0 * P.C + col0;
    step_it = P.C;
    const double ident = CT<double>::get(red_identity_bits(P.reds[0].op, RB200_T_F64));
#pragma unroll
    for (int k = 0; k < LV; ++k) cx.cacc[k] = ident;
    cx.e0 = col0 + tid;
    cx.valid = (1u << LV) - 1u;
    cx.row = 0;
    cx.staged_ok = false;
    // operands broadcast over the rows: once into the register file
    for (int h = 0; h < P.n_hoist; ++h) {
      if (P.hoist[h].is_f32_class) {
        float v[LV];
        cx.fetch_direct<float>(P.hoist[h].direct, v);
        cx.store_reg<float>(P.hoist[h].reg, v);
      } else {
        double v[LV];
        cx.fetch_direct<double>(P.hoist[h].direct, v);
        cx.store_reg<double>(P.hoist[h].reg, v);
      }
    }
  }

  auto tile_full = [&](long long it) -> bool { return P.mode == 1 || base0 + it * step_it + kStreamTile <= P.total; };
  auto issue = [&](long long it) {
    if (tid != 0) return;
    const unsigned slot = (unsigned)(it % P.depth);
    const unsigned bar = mbar_s + 8u * slot;
    const unsigned dst = smem_s + slot * P.stage_bytes;
    const long long eoff = base0 + it * step_it;
    unsigned bytes = 0;
    for (int j = 0; j < P.n_staged; ++j) bytes += (unsigned)(kStreamTile * P.staged[j].es);
    mbar_expect_tx(bar, bytes);
    for (int j = 0; j < P.n_staged; ++j)
      bulk_g2s(dst + P.staged[j].off, P.staged[j].base + eoff * P.staged[j].es, (unsigned)(kStreamTile * P.staged[j].es), bar);
  };

  if (P.n_staged > 0) {
    for (long long it = 0; it < P.depth - 1 && it < n_it; ++it)
      if (tile_full(it)) issue(it);
  }
  for (long long it = 0; it < n_it; ++it) {
    const bool full = tile_full(it);
    if (P.n_staged > 0) {
      __syncthreads();  // everyone is done with tile it-1: its stage takes tile it + depth - 1
      const long long nx = it + P.depth - 1;
      if (nx < n_it && tile_full(nx)) issue(nx);
      if (full) mbar_wait(mbar_s + 8u * (unsigned)(it % P.depth), (unsigned)((it / P.depth) & 1));
    }
    cx.staged_ok = full && P.n_staged > 0;
    cx.stage_s = smem_s + (unsigned)(it % (P.depth > 0 ? P.depth : 1)) * P.stage_bytes;
    if (P.mode == 0) {
      const long long e = base0 + it * step_it + tid;
      cx.e0 = e;
      unsigned valid = (1u << LV) - 1u;
      if (!full) {
        valid = 0;
#pragma unroll
        for (int k = 0; k < LV; ++k)
          if (e + (long long)k * kThreads < P.total) valid |= 1u << k;
      }
      cx.valid = valid;
    } else {
      cx.row = r0 + it;
    }
#pragma unroll 1
    for (int pc = 0; pc < P.n_insns; ++pc) {
      const LInsn I = P.insns[pc];
      lean_dispatch(cx, I);
    }
  }

  if (P.mode == 1) {
#pragma unroll
    for (int k = 0; k < LV; ++k) P.red_partials[split * P.C + col0 + tid + (long long)k * kThreads] = CT<double>::bits(cx.cacc[k]);
    return;
  }
  stream_finish_reductions(P, cx.racc);
}


// ---------------------------------------------------------------------------------------------
// The term form of the same op lists (rb200_terms.h): one running value per element, no dispatch tree.
// TV elements per thread per tile (tile = TV * 256 elements; element k of thread t is k*256 + t).
template <int TV> struct STermCtx {
  unsigned stage_s, hoist_s, tid;
  bool staged_ok;
  long long row, e0;
  unsigned valid;
};

// in-place arithmetic: the running value keeps its registers across the term loop (no copies at the loop's merge points)
__device__ __forceinline__ void ip_add(double& a, double b) { asm("add.rn.f64 %0, %0, %1;" : "+d"(a) : "d"(b)); }
__device__ __forceinline__ void ip_sub(double& a, double b) { asm("sub.rn.f64 %0, %0, %1;" : "+d"(a) : "d"(b)); }
__device__ __forceinline__ void ip_rsub(double& a, double b) { asm("sub.rn.f64 %0, %1, %0;" : "+d"(a) : "d"(b)); }
__device__ __forceinline__ void ip_mul(double& a, double b) { asm("mul.rn.f64 %0, %0, %1;" : "+d"(a) : "d"(b)); }
__device__ __forceinline__ void ip_add(float& a, float b) { asm("add.rn.f32 %0, %0, %1;" : "+f"(a) : "f"(b)); }
__device__ __forceinline__ void ip_sub(float& a, float b) { asm("sub.rn.f32 %0, %0, %1;" : "+f"(a) : "f"(b)); }
__device__ __forceinline__ void ip_rsub(float& a, float b) { asm("sub.rn.f32 %0, %1, %0;" : "+f"(a) : "f"(b)); }
__device__ __forceinline__ void ip_mul(float& a, float b) { asm("mul.rn.f32 %0, %0, %1;" : "+f"(a) : "f"(b)); }

template <int TV, class F>
__device__ __forceinline__ void sterm_fetch(const StreamParams& P, const STermCtx<TV>& cx, const TermStep t, F (&x)[TV]) {
  int dview = t.xidx;
  if (t.xkind == X_STAGED) {
    const StreamStaged& sv = P.staged[t.xidx];
    if (cx.staged_ok) {
      stream_lds<F, TV>(cx.stage_s + sv.off, cx.tid, sv.es == 4, x);
      return;
    }
    dview = sv.dview;  // ragged last tile: read directly
  } else if (t.xkind == X_HOIST) {
    // row-broadcast operand: this CTA's columns were copied to shared memory once
    stream_lds<F, TV>(cx.hoist_s + (unsigned)t.xidx * (TV * kThreads * 8), cx.tid, P.direct[P.thoist_direct[t.xidx]].dtype == RB200_F32, x);
    return;
  }
  const LDirect& v = P.direct[dview];
  ldirect_load<F, TV>(v, cx.row * v.s1 + cx.e0 * v.s2, (long long)kThreads * v.s2, cx.valid, x);
}

template <int TV, class F> __device__ __forceinline__ void sterm_store(const StreamParams& P, const STermCtx<TV>& cx, int dview, const F (&acc)[TV]) {
  const LDirect& v = P.direct[dview];
  const bool full = cx.valid == (TV == 32 ? 0xffffffffu : (1u << TV) - 1u);
  if (v.dtype == RB200_F32) {
    char* p = v.base + (cx.row * v.s1 + cx.e0 * v.s2) * 4;
    const long long step = (long long)kThreads * v.s2 * 4;
    if (full) {
#pragma unroll
      for (int k = 0; k < TV; ++k, p += step) stg<float>(reinterpret_cast<float*>(p), (float)acc[k]);
    } else {
#pragma unroll
      for (int k = 0; k < TV; ++k, p += step)
        if ((cx.valid >> k) & 1u) stg<float>(reinterpret_cast<float*>(p), (float)acc[k]);
    }
  } else {
    char* p = v.base + (cx.row * v.s1 + cx.e0 * v.s2) * 8;
    const long long step = (long long)kThreads * v.s2 * 8;
    if (full) {
#pragma unroll
      for (int k = 0; k < TV; ++k, p += step) stg<double>(reinterpret_cast<double*>(p), (double)acc[k]);
    } else {
#pragma unroll
      for (int k = 0; k < TV; ++k, p += step)
        if ((cx.valid >> k) & 1u) stg<double>(reinterpret_cast<double*>(p), (double)acc[k]);
    }
  }
}

// fold the thread's TV values into the accumulators of a reduction (float64 phase)
template <int TV>
__device__ __forceinline__ void sterm_reduce(const StreamParams& P, const STermCtx<TV>& cx, const TermStep t, const double (&acc)[TV], double (&cacc)[TV],
                                             double (&racc)[RB200_MAX_REDS]) {
  const int rop = t.dzl;
  if (P.mode == 1) {  // column accumulators, one per element of the thread
    if (rop == RB200_RED_ADD) {
#pragma unroll
      for (int k = 0; k < TV; ++k) ip_add(cacc[k], acc[k]);
    } else if (rop == RB200_RED_MUL) {
#pragma unroll
      for (int k = 0; k < TV; ++k) ip_mul(cacc[k], acc[k]);
    } else if (rop == RB200_RED_MIN) {
#pragma unroll
      for (int k = 0; k < TV; ++k) cacc[k] = red_combine<double>(RB200_RED_MIN, cacc[k], acc[k]);
    } else {
#pragma unroll
      for (int k = 0; k < TV; ++k) cacc[k] = red_combine<double>(RB200_RED_MAX, cacc[k], acc[k]);
    }
    return;
  }
  double x[TV];
  const bool full = cx.valid == (TV == 32 ? 0xffffffffu : (1u << TV) - 1u);
  if (full) {
#pragma unroll
    for (int k = 0; k < TV; ++k) x[k] = acc[k];
  } else {
    const double ident = CT<double>::get(red_identity_bits(rop, RB200_T_F64));
#pragma unroll
    for (int k = 0; k < TV; ++k) x[k] = ((cx.valid >> k) & 1u) ? acc[k] : ident;
  }
  double r;
  if (rop == RB200_RED_ADD) {
#pragma unroll
    for (int w = TV / 2; w > 0; w /= 2) {
#pragma unroll
      for (int k = 0; k < w; ++k) x[k] = __dadd_rn(x[k], x[k + w]);
    }
    r = x[0];
  } else {
#pragma unroll
    for (int w = TV / 2; w > 0; w /= 2) {
#pragma unroll
      for (int k = 0; k < w; ++k) x[k] = red_combine<double>(rop, x[k], x[k + w]);
    }
    r = x[0];
  }
#pragma unroll
  for (int q = 0; q < RB200_MAX_REDS; ++q)
    if (q == (int)t.sidx) racc[q] = red_combine<double>(rop, racc[q], r);
}

template <int TV, class F>
__device__ __forceinline__ void sterm_step(const StreamParams& P, const STermCtx<TV>& cx, const TermStep t, F (&acc)[TV], double (&cacc)[TV],
                                           double (&racc)[RB200_MAX_REDS]) {
  {
    if (t.kind >= TK_NEG) {
      if (t.kind == TK_NEG) {
#pragma unroll
        for (int k = 0; k < TV; ++k) acc[k] = -acc[k];
      } else if (t.kind == TK_ROUND32) {
#pragma unroll
        for (int k = 0; k < TV; ++k) acc[k] = (F)(float)acc[k];  // the value a float32 temporary would hold
      } else if (t.kind == TK_STORE) {
        sterm_store<TV, F>(P, cx, t.xidx, acc);
      } else if constexpr (sizeof(F) == 8) {
        sterm_reduce<TV>(P, cx, t, acc, cacc, racc);
      }
      return;
    }
    F w = F(0);
    if (t.flags & TF_W) w = scal_as<F>(P.scal[t.sidx]);
    if (t.kind == TK_SET) {  // straight into the running value
      if (t.xkind != X_NONE) {
        sterm_fetch<TV, F>(P, cx, t, acc);
        if (t.flags & TF_W) {
#pragma unroll
          for (int k = 0; k < TV; ++k) ip_mul(acc[k], w);
        }
      } else {
#pragma unroll
        for (int k = 0; k < TV; ++k) acc[k] = w;
      }
      return;
    }
    if (t.xkind == X_NONE) {  // acc (op) scalar
      if (t.kind == TK_MUL) {
#pragma unroll
        for (int k = 0; k < TV; ++k) ip_mul(acc[k], w);
      } else if (t.flags & TF_NEGP) {
#pragma unroll
        for (int k = 0; k < TV; ++k) ip_sub(acc[k], w);
      } else if (t.flags & TF_NEGACC) {
#pragma unroll
        for (int k = 0; k < TV; ++k) ip_rsub(acc[k], w);
      } else {
#pragma unroll
        for (int k = 0; k < TV; ++k) ip_add(acc[k], w);
      }
      return;
    }
    F p[TV];
    sterm_fetch<TV, F>(P, cx, t, p);
    if (t.flags & TF_W) {
#pragma unroll
      for (int k = 0; k < TV; ++k) ip_mul(p[k], w);
    }
    if (t.kind == TK_MUL) {
#pragma unroll
      for (int k = 0; k < TV; ++k) ip_mul(acc[k], p[k]);
    } else if (t.flags & TF_NEGP) {
#pragma unroll
      for (int k = 0; k < TV; ++k) ip_sub(acc[k], p[k]);
    } else if (t.flags & TF_NEGACC) {
#pragma unroll
      for (int k = 0; k < TV; ++k) ip_rsub(acc[k], p[k]);
    } else {
#pragma unroll
      for (int k = 0; k < TV; ++k) ip_add(acc[k], p[k]);
    }
  }
}

// the first kUnrolledSteps steps are unrolled: their descriptors sit at fixed constant-bank addresses, so the compiler
// loads and decodes them ONCE, outside the loop over tiles
constexpr int kUnrolledSteps = 6;
template <int TV, class F>
__device__ __forceinline__ void sterm_steps(const StreamParams& P, const STermCtx<TV>& cx, int s0, int s1, F (&acc)[TV], double (&cacc)[TV],
                                            double (&racc)[RB200_MAX_REDS]) {
#pragma unroll
  for (int u = 0; u < kUnrolledSteps; ++u)
    if (s0 + u < s1) sterm_step<TV, F>(P, cx, P.terms[s0 + u], acc, cacc, racc);
#pragma unroll 1
  for (int s = s0 + kUnrolledSteps; s < s1; ++s) sterm_step<TV, F>(P, cx, P.terms[s], acc, cacc, racc);
}

#ifndef RB200_STREAM_MINB8
#define RB200_STREAM_MINB8 3
#endif
template <int TV>
__global__ void __launch_bounds__(kThreads, TV == 8 ? RB200_STREAM_MINB8 : 2) stream_terms_kernel(const __grid_constant__ StreamParams P) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const unsigned smem_s = (unsigned)__cvta_generic_to_shared(smem_raw);
  const unsigned tid = threadIdx.x;
  constexpr int TILE = TV * kThreads;
  // layout: [ring: depth stages][hoisted operands: n_thoist * TILE * 8][mbarriers]
  const unsigned hoist_s = smem_s + (unsigned)P.depth * P.stage_bytes;
  const unsigned mbar_s = hoist_s + (unsigned)P.n_thoist * (TILE * 8);
  if (P.n_staged > 0 && tid == 0) {
    for (int s = 0; s < P.depth; ++s) mbar_init(mbar_s + 8u * s, 1u);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  STermCtx<TV> cx;
  cx.tid = tid;
  cx.hoist_s = hoist_s;
  double racc[RB200_MAX_REDS];
  double cacc[TV];
#pragma unroll
  for (int s = 0; s < RB200_MAX_REDS; ++s) racc[s] = 0.0;
  for (int s = 0; s < P.n_reds; ++s) {
    const double ident = CT<double>::get(red_identity_bits(P.reds[s].op, RB200_T_F64));
#pragma unroll
    for (int q = 0; q < RB200_MAX_REDS; ++q)
      if (q == s) racc[q] = ident;
  }
#pragma unroll
  for (int k = 0; k < TV; ++k) cacc[k] = 0.0;
  long long n_it, base0, step_it;  // element offset of tile `it` = base0 + it * step_it
  long long split = 0, col0 = 0, r0 = 0;
  if (P.mode == 0) {
    n_it = (P.n_tiles - (long long)blockIdx.x + gridDim.x - 1) / gridDim.x;
    base0 = (long long)blockIdx.x * TILE;
    step_it = (long long)gridDim.x * TILE;
    cx.row = 0;
  } else {
    split = blockIdx.x / (unsigned)P.n_chunks;
    const long long chunk = blockIdx.x - split * P.n_chunks;
    col0 = chunk * TILE;
    r0 = split * P.rows_per_split;
    long long r1 = r0 + P.rows_per_split;
    if (r1 > P.R) r1 = P.R;
    n_it = r1 > r0 ? r1 - r0 : 0;
    base0 = r0 * P.C + col0;
    step_it = P.C;
    const double ident = CT<double>::get(red_identity_bits(P.reds[0].op, RB200_T_F64));
#pragma unroll
    for (int k = 0; k < TV; ++k) cacc[k] = ident;
    cx.e0 = col0 + tid;
    cx.valid = TV == 32 ? 0xffffffffu : (1u << TV) - 1u;
    cx.row = 0;
    // operands broadcast over the rows: this CTA's columns once into shared memory (natural element order)
    for (int h = 0; h < P.n_thoist; ++h) {
      const LDirect& v = P.direct[P.thoist_direct[h]];
      const unsigned dst = hoist_s + (unsigned)h * (TILE * 8);
      if (v.dtype == RB200_F32) {
        const float* p = reinterpret_cast<const float*>(v.base) + col0;
        for (int e = (int)tid; e < TILE; e += kThreads) lean_sts<float>(dst + (unsigned)e * 4u, ldg<float>(p + e));
      } else {
        const double* p = reinterpret_cast<const double*>(v.base) + col0;
        for (int e = (int)tid; e < TILE; e += kThreads) lean_sts<double>(dst + (unsigned)e * 8u, ldg<double>(p + e));
      }
    }
  }
  __syncthreads();

  auto tile_full = [&](long long it) -> bool { return P.mode == 1 || base0 + it * step_it + TILE <= P.total; };
  auto issue = [&](long long it, int slot) {
    if (tid != 0) return;
    const unsigned bar = mbar_s + 8u * (unsigned)slot;
    const unsigned dst = smem_s + (unsigned)slot * P.stage_bytes;
    const long long eoff = base0 + it * step_it;
    mbar_expect_tx(bar, P.stage_bytes);
    for (int j = 0; j < P.n_staged; ++j)
      bulk_g2s(dst + P.staged[j].off, P.staged[j].base + eoff * P.staged[j].es, (unsigned)(TILE * P.staged[j].es), bar);
  };
  int islot = 0;  // ring slot of the next tile to request
  if (P.n_staged > 0) {
    for (long long it = 0; it < P.depth - 1 && it < n_it; ++it) {
      if (tile_full(it)) issue(it, islot);
      islot = islot + 1 >= P.depth ? 0 : islot + 1;
    }
  }
  int slot = 0;
  unsigned par = 0;
  for (long long it = 0; it < n_it; ++it) {
    const bool full = tile_full(it);
    if (P.n_staged > 0) {
      __syncthreads();  // everyone is done with tile it-1: its stage takes tile it + depth - 1
      const long long nx = it + P.depth - 1;
      if (nx < n_it) {
        if (tile_full(nx)) issue(nx, islot);
        islot = islot + 1 >= P.depth ? 0 : islot + 1;
      }
      if (full) {
        mbar_wait(mbar_s + 8u * (unsigned)slot, (par >> slot) & 1u);
        par ^= 1u << slot;
      }
    }
    cx.staged_ok = full && P.n_staged > 0;
    cx.stage_s = smem_s + (unsigned)slot * P.stage_bytes;
    slot = slot + 1 >= P.depth ? 0 : slot + 1;
    if (P.mode == 0) {
      const long long e = base0 + it * step_it + tid;
      cx.e0 = e;
      unsigned valid = TV == 32 ? 0xffffffffu : (1u << TV) - 1u;
      if (!full) {
        valid = 0;
#pragma unroll
        for (int k = 0; k < TV; ++k)
          if (e + (long long)k * kThreads < P.total) valid |= 1u << k;
      }
      cx.valid = valid;
    } else {
      cx.row = r0 + it;
    }
    if (P.n32 > 0) {
      float a32[TV];
      sterm_steps<TV, float>(P, cx, 0, P.n32, a32, cacc, racc);
      if (P.n_terms > P.n32) {
        double a64[TV];
#pragma unroll
        for (int k = 0; k < TV; ++k) a64[k] = (double)a32[k];
        sterm_steps<TV, double>(P, cx, P.n32, P.n_terms, a64, cacc, racc);
      }
    } else {
      double a64[TV];
      sterm_steps<TV, double>(P, cx, 0, P.n_terms, a64, cacc, racc);
    }
  }

  if (P.mode == 1) {
#pragma unroll
    for (int k = 0; k < TV; ++k) P.red_partials[split * P.C + col0 + tid + (long long)k * kThreads] = CT<double>::bits(cacc[k]);
    return;
  }
  stream_finish_reductions(P, racc);
}

// =============================================================================================
// host side

// the view tables; view_kind / view_arg / store_arg: how lean_translate addresses each view
static void stream_views(const rb200_fused_op* op, StreamParams& P, bool column_mode, long long row_len, int* view_kind, int* view_arg, int* store_arg) {
  // staged: read views that are contiguous along the iteration (and, in column mode, over the rows) with 16-byte
  // aligned tiles; everything else direct
  const ViewUse use = view_use(op);
  unsigned off = 0;
  for (int v = 0; v < op->n_views; ++v) {
    const rb200_view& vw = op->views[v];
    const int es = vw.dtype == RB200_F64 ? 8 : 4;
    LDirect& d = P.direct[P.n_direct];
    d.base = (char*)vw.base;
    d.s0 = 0;
    d.s1 = column_mode ? vw.stride[0] : 0;
    d.s2 = column_mode ? vw.stride[1] : vw.stride[0];
    d.dtype = vw.dtype;
    view_kind[v] = L_DIRECT;
    view_arg[v] = store_arg[v] = P.n_direct;
    const bool contiguous = d.s2 == 1 && (!column_mode || d.s1 == row_len);
    const bool aligned = (((uintptr_t)vw.base) & 15u) == 0 && (!column_mode || (row_len * es) % 16 == 0);
    if (use.read[v] && contiguous && aligned && P.n_staged < kStreamMaxStaged) {
      StreamStaged& s = P.staged[P.n_staged];
      s.base = (const char*)vw.base;
      s.es = es;
      s.dview = P.n_direct;
      s.off = off;
      off += (unsigned)(kStreamTile * es);
      view_kind[v] = L_STAGED;
      view_arg[v] = P.n_staged;
      ++P.n_staged;
    }
    ++P.n_direct;
  }
  P.stage_bytes = off;
  P.n_insns = op->n_insns;
  P.n_regs = op->n_regs;
  for (int i = 0; i < op->n_scalars; ++i) P.scal[i] = op->scalars[i];
}

// byte offsets of the staged views inside a stage for tiles of tv * 256 elements
static void stream_layout(StreamParams& P) {
  unsigned off = 0;
  for (int j = 0; j < P.n_staged; ++j) {
    P.staged[j].off = off;
    off += (unsigned)(P.tv * kThreads * P.staged[j].es);
  }
  P.stage_bytes = off;
}

// shared-memory budget: ring depth from what is left after the register file / hoisted operands.  0: does not fit.
static size_t stream_smem(StreamParams& P) {
  const size_t tile = (size_t)P.tv * kThreads;
  const size_t regs = P.n_terms > 0 ? (size_t)P.n_thoist * tile * 8 : (size_t)(P.n_regs + P.n_hoist) * LV * kThreads * 8;
  const size_t budget = P.n_terms > 0 ? 70 * 1024 : 100 * 1024;  // (term kernel: 3 CTAs per SM)
  if (regs + 1024 > budget) return 0;
  int depth = 0;
  if (P.n_staged > 0) {
    depth = (int)((budget - regs - 256) / P.stage_bytes);
    if (depth > 8) depth = 8;
    if (depth < 2) return 0;
  }
  P.depth = depth;
  return (size_t)depth * P.stage_bytes + regs + (size_t)(depth > 0 ? depth : 1) * 8 + 16;
}

bool plan_stream(const rb200_fused_op* op, int sms, int n_split, bool use_terms, bool use_mapred, StreamPlan& T) {
  StreamParams& P = T.P;
  memset(&T, 0, sizeof(T));
  const bool column = op->n_axis_red_dims != 0;
  if (!column) {
    if (op->ndim != 1) return false;
    if (!lean_vocabulary_only(op, true)) return false;
    for (int s = 0; s < op->n_reds; ++s) {
      if (op->reds[s].ctype != RB200_T_F64) return false;
      if (op->reds[s].out_dtype != RB200_F64 && op->reds[s].out_dtype != RB200_F32) return false;
    }
    P.mode = 0;
    P.total = op->itershape[0];
  } else {
    if (op->ndim != 2 || op->n_axis_red_dims != 1 || op->n_reds != 1) return false;
    if (!lean_vocabulary_only(op, true)) return false;
    if (op->reds[0].ctype != RB200_T_F64) return false;
    const long long R = op->itershape[0], C = op->itershape[1];
    if (C % (LV * kThreads) != 0 || R < 2) return false;
    for (int i = 0; i < op->n_insns; ++i)
      if (op->insns[i].st_view != RB200_NOSTORE) return false;
    for (int v = 0; v < op->n_views; ++v) {
      const rb200_view& vw = op->views[v];
      if (vw.stride[1] != 1 || !(vw.stride[0] == C || vw.stride[0] == 0)) return false;
    }
    P.mode = 1;
    P.R = R;
    P.C = C;
    P.total = R * C;
  }
  P.tv = LV;
  int view_kind[RB200_MAX_VIEWS], view_arg[RB200_MAX_VIEWS], store_arg[RB200_MAX_VIEWS];
  stream_views(op, P, column, P.C, view_kind, view_arg, store_arg);
  lean_translate(op, op->insns, view_kind, view_arg, store_arg, P.insns);
  // ---- the term form first
  TermBuild tb;
  tb.n_regs = P.n_regs;
  tb.direct = P.direct;
  tb.stream = true;
  tb.staged_fill = [](void*, int, int, TermStep*) -> bool { return true; };
  tb.ctx = nullptr;
  int out_view = -1;
  if (use_terms && build_terms(tb, P.insns, P.n_insns, P.terms, kMaxTerms, &P.n_terms, &P.n32, &out_view)) {
    // ---- one contiguous source, scalar map, one reduction: the map + reduce kernels (no staging, no interpretation)
    auto src_of = [](void* ctx, const TermStep& t) -> MrSource {
      const StreamParams* Q = (const StreamParams*)ctx;
      MrSource r = {nullptr, 0, false};
      const LDirect* d = nullptr;
      if (t.xkind == X_STAGED) d = &Q->direct[Q->staged[t.xidx].dview];
      else if (t.xkind == X_DIRECT) d = &Q->direct[t.xidx];
      if (!d || d->s2 != 1) return r;
      if (Q->mode == 1 && !(d->s1 == Q->C || d->s1 == 0)) return r;
      r.base = d->base;
      r.f32 = d->dtype == RB200_F32;
      r.row_broadcast = Q->mode == 1 && d->s1 == 0;
      return r;
    };
    if (use_mapred && op->n_reds == 1 && mapred_try(P.mode, P.terms, P.n_terms, P.n32, P.scal, src_of, &P, &T.mr) == 0) {
      MrParams& M = T.mr;
      const int vec = M.src_f32 ? 4 : 2;
      bool ok = true;
      if (!column) {
        M.total = P.total;
        bind_reds(op, &M.red);
        bind_red_scratch(op, &M.red_counter, &M.red_partials);
        long long blocks = (P.total / (vec * 4) + kThreads - 1) / kThreads;
        long long cap = (long long)sms * 8;
        if (cap > kRedScratchPartials) cap = kRedScratchPartials;
        if (blocks > cap) blocks = cap;
        if (blocks < 1) blocks = 1;
        T.blocks = blocks;
      } else {
        const long long chunk = (long long)kThreads * vec;
        if (P.C % chunk != 0 || (P.C * (M.src_f32 ? 4 : 8)) % 16 != 0) ok = false;
        if (ok) {
          M.R = P.R;
          M.C = P.C;
          M.n_chunks = (int)(P.C / chunk);
          const int eff = row_split((long long)sms * 8, M.n_chunks, n_split, P.R);
          M.n_split = eff;
          M.rows_per_split = (P.R + eff - 1) / eff;
          M.red_partials = (u64*)op->red_scratch;
          T.eff = eff;
          T.blocks = (long long)eff * M.n_chunks;
        }
      }
      if (ok) {
        T.use_mr = true;
        T.smem = 0;
        return true;
      }
    }
    stream_layout(P);
    if (column) {
      // row-broadcast direct operands: one copy per CTA in shared memory
      for (int i = 0; i < P.n_terms; ++i) {
        TermStep& t = P.terms[i];
        if (t.xkind != X_DIRECT || P.direct[t.xidx].s1 != 0 || P.direct[t.xidx].s2 != 1) continue;
        int h = -1;
        for (int q = 0; q < P.n_thoist; ++q)
          if (P.thoist_direct[q] == t.xidx) h = q;
        if (h < 0 && P.n_thoist < kStreamMaxStaged) {
          h = P.n_thoist++;
          P.thoist_direct[h] = t.xidx;
        }
        if (h >= 0) {
          t.xkind = X_HOIST;
          t.xidx = (unsigned char)h;
        }
      }
    }
  } else {
    P.n_terms = 0;
    if (column) {
      // the lean kernel: row-broadcast operands fetched in one class move into the register file, so the list is
      // translated again from a hoisted copy (the term form above reads them from the direct views)
      rb200_insn insns[RB200_MAX_INSNS];
      memcpy(insns, op->insns, sizeof(rb200_insn) * op->n_insns);
      int view[kStreamMaxStaged], reg[kStreamMaxStaged], cls[kStreamMaxStaged];
      P.n_hoist = hoist_row_broadcast(op, insns, P.n_regs, 255, kStreamMaxStaged, view, reg, cls);
      for (int j = 0; j < P.n_hoist; ++j) P.hoist[j] = {view[j], reg[j], cls[j] == RB200_T_F32};
      lean_translate(op, insns, view_kind, view_arg, store_arg, P.insns);
    }
  }
  T.smem = stream_smem(P);
  if (T.smem == 0) return false;
  const long long tile = (long long)P.tv * kThreads;
  P.n_reds = op->n_reds;
  bind_reds(op, P.reds);
  if (!column) {
    P.n_tiles = (P.total + tile - 1) / tile;
    if (op->n_reds > 0) bind_red_scratch(op, &P.red_counter, &P.red_partials);
    long long blocks = P.n_tiles;
    long long cap = (long long)sms * ((P.n_terms > 0 && T.smem <= 72 * 1024) ? RB200_STREAM_MINB8 : 2);
    if (op->n_reds > 0 && cap > kRedScratchPartials) cap = kRedScratchPartials;
    if (blocks > cap) blocks = cap;
    T.blocks = blocks;
  } else {
    P.n_chunks = (int)(P.C / tile);
    const int per_sm = (P.n_terms > 0 && T.smem <= 72 * 1024) ? RB200_STREAM_MINB8 : 2;
    if (P.n_chunks > sms * per_sm) return false;
    const int eff = row_split((long long)sms * per_sm, P.n_chunks, n_split, P.R);
    P.n_split = eff;
    P.rows_per_split = (P.R + eff - 1) / eff;
    P.red_partials = (u64*)op->red_scratch;
    T.eff = eff;
    T.blocks = (long long)eff * P.n_chunks;
  }
  return true;
}

std::string describe_stream(const StreamPlan& T) {
  const StreamParams& P = T.P;
  char buf[320];
  if (T.use_mr) {
    snprintf(buf, sizeof(buf), "kernel=mapred mode=%s source=%s ops=%d(f32:%d) broadcast_operand=%d reduction=%d loads=128bit ctas=%lld", P.mode == 0 ? "global" : "columns",
             T.mr.src_f32 ? "f32" : "f64", T.mr.n32 + T.mr.n64, T.mr.n32, T.mr.vsrc ? 1 : 0, T.mr.redop, T.blocks);
    return buf;
  }
  snprintf(buf, sizeof(buf),
           "kernel=%s mode=%s staged_views=%d ring_depth=%d stage_bytes=%u direct_views=%d hoisted=%d lean_insns=%d terms=%d(f32:%d) tile=%d reds=%d "
           "ctas=%lld smem=%zu",
           P.n_terms > 0 ? "stream_terms" : "stream", P.mode == 0 ? "elementwise" : "columns", P.n_staged, P.depth, P.stage_bytes, P.n_direct,
           P.n_terms > 0 ? P.n_thoist : P.n_hoist, P.n_insns, P.n_terms, P.n32, P.tv * kThreads, P.n_reds, T.blocks, T.smem);
  return buf;
}

cudaError_t launch_stream(const StreamPlan& T, cudaStream_t stream) {
  if (T.use_mr) return mapred_launch(T.mr, (unsigned)T.blocks, stream);
  static const bool attrs = []() {  // (set once, thread-safe)
    cudaFuncSetAttribute(stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 101 * 1024);
    cudaFuncSetAttribute(stream_terms_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 101 * 1024);
    return true;
  }();
  (void)attrs;
  if (T.P.n_terms > 0) stream_terms_kernel<8><<<(unsigned)T.blocks, kThreads, T.smem, stream>>>(T.P);
  else stream_kernel<<<(unsigned)T.blocks, kThreads, T.smem, stream>>>(T.P);
  return cudaGetLastError();
}

}  // namespace rb200
