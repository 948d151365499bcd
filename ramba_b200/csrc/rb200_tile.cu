// rb200_tile.cu — K2: the shifted-view stencil / N-d float arithmetic kernel (sm_90a).
//
// What it stands for in the reference: the "locally optimised" generated kernel for fused ops whose operands are
// shifted slice views of one array - one base argument per array plus per-view offsets, body
//   acc = U[o1_0+i0, o1_1+i1, o1_2+i2] + U[o2_0+i0, ...] + ... ; V[index] = acc - c*U[...]
// (ramba/ramba.py:8146-8188, SURVEY §8a "textbook shifted-pointer stencil"), executed by RemoteState.run_deferred_ops
// (ramba/ramba.py:3758-3780).
//
// Design (H100):
//   * The iteration box (2-D or 3-D after host-side collapsing) is cut into tiles of TY x TX = 2048 outputs
//     (256 threads x 8); a CTA takes a tile column and MARCHES along the outermost dim, ZC planes per work item.
//   * The read-only views that are shifted copies of each other (same dtype, same strides, base offsets that decompose
//     into small per-dim shifts) form the STAGED GROUP: for every plane the CTA needs, ONE box of
//     (TY + halo_y) x (TX + halo_x) elements is copied global -> shared by the TMA engine
//     (cp.async.bulk.tensor, SASS UTMALDG; completion on an mbarrier), into a ring of halo_z + 2 planes, one plane
//     ahead of the computation.  Every element of the source array is read from HBM once per (tile column, plane);
//     the 7 (or 5, 9, 13, 25...) neighbour reads of the op list become shared-memory loads at an offset known per
//     instruction.  When the source does not meet the TMA rules (16-byte aligned strides) or the box could leave the
//     shard buffer, the same box is filled by per-thread cp.async (LDGSTS) with bounds predicates.
//   * Everything else the op list touches (other operands, the destination) is addressed directly in global memory,
//     coalesced along x.
//   * The op list itself runs on the lean machine (rb200_lean.cuh): same order, same classes, same roundings as the
//     general interpreter.
// Grid: persistent, 2 CTAs per SM.  Bound: HBM (read the source once + write the destination once).
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdio.h>
#include <string.h>

#include <string>

#include "rb200_launch.h"
#include "rb200_lean.cuh"
#include "rb200_plan.h"
#include "rb200_terms.h"
#include "rb200_tile.h"

namespace rb200 {

__device__ __forceinline__ void tma_load_3d(unsigned sdst, const CUtensorMap* tmap, int c0, int c1, int c2, unsigned mbar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(sdst),
      "l"(tmap), "r"(mbar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void cp_async_mbar_arrive(unsigned mbar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(mbar) : "memory");
}

// ask for plane `pz` (halo coordinates) of the staged group into ring slot `slot`
template <class TE>
__device__ __forceinline__ void tile_request(const TileParams& P, const CUtensorMap* tmap, unsigned smem_s, unsigned mbar_s, unsigned slot, long long x0,
                                             long long y0, long long pz, unsigned tid) {
  const unsigned bar = mbar_s + 8u * slot;
  const unsigned dst = smem_s + slot * P.plane_bytes;
  if (P.use_tma) {
    if (tid == 0) {
      mbar_expect_tx(bar, (unsigned)(kTilePX * P.PY * (int)sizeof(TE)));
      tma_load_3d(dst, tmap, (int)x0 + P.tma_shift, (int)y0, (int)pz, bar);
    }
  } else {
    // rows of the box by warps, elements by lanes; out-of-range elements are zero-filled
    const int lane = (int)(tid & 31u), warp = (int)(tid >> 5);
    const long long Xh = P.X + P.hx, Yh = P.Y + P.hy, Zh = P.Z + P.hz;
    for (int py = warp; py < P.PY; py += kThreads / 32) {
      const long long gy = y0 + py;
      const TE* row = reinterpret_cast<const TE*>(P.gcorner) + pz * P.gs0 + gy * P.gs1 + x0;
      const unsigned drow = dst + (unsigned)(py * kTilePX * (int)sizeof(TE));
      const bool row_ok = gy < Yh && pz >= 0 && pz < Zh;
      for (int px = lane; px < kTilePX; px += 32) {
        const TE* src = row + px;
        const bool ok = row_ok && (x0 + px) < Xh && (const char*)src >= P.safe_lo && (const char*)(src + 1) <= P.safe_hi;
        if constexpr (sizeof(TE) == 8) cp_async8(drow + px * 8u, ok ? (const void*)src : (const void*)P.safe_lo, ok);
        else cp_async4(drow + px * 4u, ok ? (const void*)src : (const void*)P.safe_lo, ok);
      }
    }
    cp_async_mbar_arrive(bar);
  }
}

template <class TE> struct TileCtx : LeanRegs {
  const TileParams& P;
  unsigned ring_s;  // shared-window address of the plane ring
  unsigned tb0;     // byte offset of this thread's element k = 0 inside a plane, before the operand's own (dy, dx) offset
  static constexpr unsigned kstep = (unsigned)(kTileRY * kTilePX * sizeof(TE));  // byte step between elements k and k+1 inside a plane
  int fb;           // ring slot holding plane (z - hz_lo)
  long long z, gy0, gx;
  unsigned valid;
  __device__ __forceinline__ TileCtx(const TileParams& p) : P(p) {}

  template <class F> __device__ __forceinline__ void fetch(int kind, int arg, F (&out)[LV]) {
    switch (kind) {
      case L_STAGED: {
        const TileStagedOp t = P.staged[arg];
        int slot = fb + t.dzl;
        if (slot >= P.D) slot -= P.D;
        const unsigned addr = ring_s + (unsigned)slot * P.plane_bytes + t.off + tb0;
#pragma unroll
        for (int k = 0; k < LV; ++k) out[k] = (F)lean_lds<TE>(addr + k * kstep);
      } break;
      case L_DIRECT: {
        const LDirect& v = P.direct[arg];
        ldirect_load<F, LV>(v, z * v.s0 + gy0 * v.s1 + gx * v.s2, (long long)kTileRY * v.s1, valid, out);
      } break;
      case L_REG: fetch_reg<F>(arg, out); break;
      case L_SCAL: fetch_scal<F>(P.scal[arg], out); break;
      default: fetch_acc<F>(out);  // L_ACC
    }
  }
  template <class F> __device__ __forceinline__ int chain_fetch(int step, F (&out)[LV]) {
    const LChainStep cs = P.chain[step];
    const TileStagedOp t = P.staged[cs.staged];
    int slot = fb + t.dzl;
    if (slot >= P.D) slot -= P.D;
    const unsigned addr = ring_s + (unsigned)slot * P.plane_bytes + t.off + tb0;
#pragma unroll
    for (int k = 0; k < LV; ++k) out[k] = (F)lean_lds<TE>(addr + k * kstep);
    return cs.op;
  }
  template <class F> __device__ __forceinline__ void store_view(int arg, const F (&r)[LV]) {
    const LDirect& v = P.direct[arg];
    ldirect_store<F, LV>(v, z * v.s0 + gy0 * v.s1 + gx * v.s2, (long long)kTileRY * v.s1, valid, r);
  }
  template <class F> __device__ __forceinline__ void reduce(int, int, const F (&)[LV]) {}  // (no reductions in this kernel)
};

template <class TE>
__global__ void __launch_bounds__(kThreads, 2) stencil_tile_kernel(const __grid_constant__ TileParams P, const __grid_constant__ CUtensorMap tmap) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const unsigned smem_s = (unsigned)__cvta_generic_to_shared(smem_raw);
  const unsigned tid = threadIdx.x;
  // layout: [ring: D planes][spill registers: n_regs * LV * 256 * 8][mbarriers: D * 8]
  const unsigned ring_bytes = (unsigned)P.D * P.plane_bytes;
  const unsigned regs_s = smem_s + ring_bytes;
  const unsigned mbar_s = regs_s + (unsigned)P.n_regs * (LV * kThreads * 8);
  if (P.has_group && tid == 0) {
    for (int s = 0; s < P.D; ++s) mbar_init(mbar_s + 8u * s, P.use_tma ? 1u : (unsigned)kThreads);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  TileCtx<TE> cx(P);
  cx.ring_s = smem_s;
  cx.reg_s = regs_s + tid * 8u;
  const int x = (int)(tid & (unsigned)(kTileTX - 1));
  const int yrow = (int)(tid >> kTileLogTX);
  cx.tb0 = (unsigned)((yrow * kTilePX + x) * (int)sizeof(TE));  // (the halo offsets are part of every staged operand's `off`)
  const int hz_hi = P.hz - P.hz_lo;
  unsigned fills = 0;  // planes this CTA has requested so far (slot = fills % D, parity = (fills / D) & 1)

  for (long long item = blockIdx.x; item < P.n_items; item += gridDim.x) {
    const int tx = (int)(item % P.nxt);
    const long long r1 = item / P.nxt;
    const int ty = (int)(r1 % P.nyt);
    const long long zc = r1 / P.nyt;
    const long long x0 = (long long)tx * kTileTX, y0 = (long long)ty * kTileTY;
    const long long zb = zc * P.ZC;
    long long ze = zb + P.ZC;
    if (ze > P.Z) ze = P.Z;
    cx.gx = x0 + x;
    cx.gy0 = y0 + yrow;
    unsigned valid = 0;
    if (cx.gx < P.X) {
#pragma unroll
      for (int k = 0; k < LV; ++k)
        if (cx.gy0 + (long long)k * kTileRY < P.Y) valid |= 1u << k;
    }
    cx.valid = valid;

    // request plane `pz` of the group (pz in halo coordinates: 0 = iteration z - hz_lo of z = 0)
    auto request = [&](long long pz) {
      tile_request<TE>(P, &tmap, smem_s, mbar_s, fills % (unsigned)P.D, x0, y0, pz, tid);
      ++fills;
    };

    unsigned fill0 = fills;  // fill index of plane zb (halo coordinate zb)
    if (P.has_group) {
      __syncthreads();  // every thread is done with the planes of the previous item
      for (int p = 0; p < P.hz + P.prefetch && p < (int)(ze - zb) + P.hz; ++p) request(zb + p);
    }
    for (long long z = zb; z < ze; ++z) {
      if (P.has_group) {
        const unsigned newest = fill0 + (unsigned)(z - zb) + (unsigned)P.hz;  // plane z + hz_hi
        if (z == zb) {
          // first plane of an item: the older planes of the prologue have their own barriers, and bulk copies may
          // complete out of order
          for (unsigned f = fill0; f < newest; ++f) mbar_wait(mbar_s + 8u * (f % (unsigned)P.D), (f / (unsigned)P.D) & 1u);
        }
        mbar_wait(mbar_s + 8u * (newest % (unsigned)P.D), (newest / (unsigned)P.D) & 1u);
        __syncthreads();  // plane z - 1 - hz_lo is free now: its slot takes the plane after the newest
        if (z + P.prefetch < ze) request(z + P.hz + P.prefetch);
        cx.fb = (int)((fill0 + (unsigned)(z - zb)) % (unsigned)P.D);
      }
      cx.z = z;
#pragma unroll 1
      for (int pc = 0; pc < P.n_insns; ++pc) {
        const LInsn I = P.insns[pc];
        lean_dispatch(cx, I);
      }
    }
  }
  (void)hz_hi;
}


// ---------------------------------------------------------------------------------------------
template <class TE, int TV> struct TermCtx {
  unsigned tb0;      // byte offset of element k = 0 of this thread inside a plane
  unsigned table_s;  // shared-window address of the per-plane operand table (one 32-bit plane address per term)
  long long z, gy0, gx;
  unsigned valid;
};

template <class TE, int TV, class F>
__device__ __forceinline__ void term_fetch(const TileParams& P, const TermCtx<TE, TV>& cx, const TermStep t, int s, F (&x)[TV]) {
  constexpr unsigned kstep = (unsigned)(kTileRY * kTilePX * sizeof(TE));
  if (t.xkind == X_STAGED) {
    const unsigned addr = lds32(cx.table_s + 4u * (unsigned)s) + cx.tb0;
#pragma unroll
    for (int k = 0; k < TV; ++k) x[k] = (F)lean_lds<TE>(addr + k * kstep);
  } else {
    const LDirect& v = P.direct[t.xidx];
    ldirect_load<F, TV>(v, cx.z * v.s0 + cx.gy0 * v.s1 + cx.gx * v.s2, (long long)kTileRY * v.s1, cx.valid, x);
  }
}

template <class TE, int TV, class F>
__device__ __forceinline__ void term_steps(const TileParams& P, const TermCtx<TE, TV>& cx, int s0, int s1, F (&acc)[TV]) {
  constexpr unsigned kstep = (unsigned)(kTileRY * kTilePX * sizeof(TE));
  int s = s0;
#pragma unroll 1
  while (s < s1) {
    const int run = P.term_run[s];
    if (run > 0) {
      // the neighbour sum: `run` consecutive terms acc = acc (+|-) x over staged operands, nothing to decode per term
      // but the operand's plane address (one broadcast shared-memory load)
      const bool neg = (P.terms[s].flags & TF_NEGP) != 0;
      const int e = s + run;
      if (!neg) {
#pragma unroll 1
        for (; s < e; ++s) {
          const unsigned addr = lds32(cx.table_s + 4u * (unsigned)s) + cx.tb0;
#pragma unroll
          for (int k = 0; k < TV; ++k) acc[k] = l_add<F>(acc[k], (F)lean_lds<TE>(addr + k * kstep));
        }
      } else {
#pragma unroll 1
        for (; s < e; ++s) {
          const unsigned addr = lds32(cx.table_s + 4u * (unsigned)s) + cx.tb0;
#pragma unroll
          for (int k = 0; k < TV; ++k) acc[k] = l_sub<F>(acc[k], (F)lean_lds<TE>(addr + k * kstep));
        }
      }
      continue;
    }
    const TermStep t = P.terms[s];
    if (t.kind == TK_NEG) {
#pragma unroll
      for (int k = 0; k < TV; ++k) acc[k] = -acc[k];
      ++s;
      continue;
    }
    F p[TV];
    if (t.xkind != X_NONE) {
      term_fetch<TE, TV, F>(P, cx, t, s, p);
      if (t.flags & TF_W) {
        const F w = scal_as<F>(P.scal[t.sidx]);
#pragma unroll
        for (int k = 0; k < TV; ++k) p[k] = l_mul<F>(p[k], w);
      }
    } else {
      const F w = scal_as<F>(P.scal[t.sidx]);
#pragma unroll
      for (int k = 0; k < TV; ++k) p[k] = w;
    }
    if (t.kind == TK_ADD) {
      if (t.flags & TF_NEGP) {
#pragma unroll
        for (int k = 0; k < TV; ++k) acc[k] = l_sub<F>(acc[k], p[k]);
      } else if (t.flags & TF_NEGACC) {
#pragma unroll
        for (int k = 0; k < TV; ++k) acc[k] = l_sub<F>(p[k], acc[k]);
      } else {
#pragma unroll
        for (int k = 0; k < TV; ++k) acc[k] = l_add<F>(acc[k], p[k]);
      }
    } else if (t.kind == TK_MUL) {
#pragma unroll
      for (int k = 0; k < TV; ++k) acc[k] = l_mul<F>(acc[k], p[k]);
    } else {  // TK_SET
#pragma unroll
      for (int k = 0; k < TV; ++k) acc[k] = p[k];
    }
    ++s;
  }
}

// TV elements per thread per plane: tile = 128 columns x 2*TV rows
template <class TE, int TV>
#ifndef RB200_TERMS_MINB
#define RB200_TERMS_MINB 3
#endif
__global__ void __launch_bounds__(kThreads, (TV == 8 && sizeof(TE) == 4) ? RB200_TERMS_MINB : 2) stencil_terms_kernel(const __grid_constant__ TileParams P, const __grid_constant__ CUtensorMap tmap) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const unsigned smem_s = (unsigned)__cvta_generic_to_shared(smem_raw);
  const unsigned tid = threadIdx.x;
  // layout: [ring: D planes][operand table, double buffered by plane parity: 2 * kTileMaxTerms * 4][mbarriers: D * 8]
  const unsigned table_s = smem_s + (unsigned)P.D * P.plane_bytes;
  const unsigned mbar_s = table_s + 2u * kTileMaxTerms * 4u;
  if (P.has_group && tid == 0) {
    for (int s = 0; s < P.D; ++s) mbar_init(mbar_s + 8u * s, P.use_tma ? 1u : (unsigned)kThreads);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  TermCtx<TE, TV> cx;
  cx.table_s = table_s;
  const int x = (int)(tid & (unsigned)(kTileTX - 1));
  const int yrow = (int)(tid >> kTileLogTX);
  cx.tb0 = (unsigned)((yrow * kTilePX + x) * (int)sizeof(TE));
  const int D = P.D, hz = P.hz;
  constexpr int TY = TV * kTileRY;
  int rq = 0;        // ring slot of the next plane to request
  unsigned par = 0;  // bit s: parity of the next completion to wait for on slot s
  // this thread's entry of the operand table (threads 0 .. n_terms-1): static part
  unsigned my_off = 0;
  int my_dzl = -1;
  if ((int)tid < P.n_terms && P.terms[tid].xkind == X_STAGED) {
    my_off = P.terms[tid].off;
    my_dzl = P.terms[tid].dzl;
  }

  for (long long item = blockIdx.x; item < P.n_items; item += gridDim.x) {
    const int tx = (int)(item % P.nxt);
    const long long r1 = item / P.nxt;
    const int ty = (int)(r1 % P.nyt);
    const long long zc = r1 / P.nyt;
    const long long x0 = (long long)tx * kTileTX, y0 = (long long)ty * TY;
    const long long zb = zc * P.ZC;
    long long ze = zb + P.ZC;
    if (ze > P.Z) ze = P.Z;
    cx.gx = x0 + x;
    cx.gy0 = y0 + yrow;
    unsigned valid = 0;
    if (cx.gx < P.X) {
#pragma unroll
      for (int k = 0; k < TV; ++k)
        if (cx.gy0 + (long long)k * kTileRY < P.Y) valid |= 1u << k;
    }
    cx.valid = valid;
    // output: address of this thread's element k = 0 of plane zb, advanced by one plane per iteration
    const LDirect& ov = P.direct[P.out_view];
    const int oes = ov.dtype == RB200_F64 ? 8 : 4;
    char* optr = ov.base + (zb * ov.s0 + cx.gy0 * ov.s1 + cx.gx * ov.s2) * oes;
    const long long ostep = (long long)kTileRY * ov.s1 * oes, oplane = ov.s0 * oes;
    int cur = rq;  // slot of plane (zb - hz_lo)
    if (P.has_group) {
      __syncthreads();  // every thread is done with the planes of the previous item
      for (int p = 0; p < hz + P.prefetch && p < (int)(ze - zb) + hz; ++p) {
        tile_request<TE>(P, &tmap, smem_s, mbar_s, (unsigned)rq, x0, y0, zb + p, tid);
        rq = rq + 1 == D ? 0 : rq + 1;
      }
    }
    for (long long z = zb; z < ze; ++z) {
      if (P.has_group) {
        int sl = cur;
        if (z == zb) {
          // first plane of an item: every plane of the prologue has its own barrier (bulk copies may complete out of order)
          for (int p = 0; p < hz; ++p) {
            mbar_wait(mbar_s + 8u * (unsigned)sl, (par >> sl) & 1u);
            par ^= 1u << sl;
            sl = sl + 1 == D ? 0 : sl + 1;
          }
        } else {
          sl = cur + hz;
          if (sl >= D) sl -= D;
        }
        mbar_wait(mbar_s + 8u * (unsigned)sl, (par >> sl) & 1u);  // the newest plane, z + hz_hi
        par ^= 1u << sl;
        if (my_dzl >= 0) {  // where this plane's copy of my term's operand starts
          int q = cur + my_dzl;
          if (q >= D) q -= D;
          // (two tables: a thread that is still computing plane z - 1 reads the other one)
          asm volatile("st.shared.u32 [%0], %1;" ::"r"(table_s + ((unsigned)z & 1u) * (kTileMaxTerms * 4u) + 4u * tid),
                       "r"(smem_s + (unsigned)q * P.plane_bytes + my_off)
                       : "memory");
        }
        __syncthreads();  // plane z - 1 - hz_lo is free now: its slot takes the plane after the newest; the table is visible
        if (z + P.prefetch < ze) {
          tile_request<TE>(P, &tmap, smem_s, mbar_s, (unsigned)rq, x0, y0, z + hz + P.prefetch, tid);
          rq = rq + 1 == D ? 0 : rq + 1;
        }
        cur = cur + 1 == D ? 0 : cur + 1;
      }
      cx.z = z;
      cx.table_s = table_s + ((unsigned)z & 1u) * (kTileMaxTerms * 4u);
      if (P.n32 > 0) {
        if constexpr (sizeof(TE) == 4) {
          constexpr unsigned kstep = (unsigned)(kTileRY * kTilePX * sizeof(TE));
          float a32[TV];
          term_steps<TE, TV, float>(P, cx, 0, P.n32, a32);
          if (P.fast_tail) {
            // the usual end of a stencil: ONE weighted staged term in float64 (`acc -+ w*x`), then the store
            const TermStep t = P.terms[P.n32];
            const double w = __longlong_as_double((long long)P.scal[t.sidx]);
            const unsigned addr = lds32(cx.table_s + 4u * (unsigned)P.n32) + cx.tb0;
            double r[TV];
            if (t.flags & TF_NEGP) {
#pragma unroll
              for (int k = 0; k < TV; ++k) r[k] = __dsub_rn((double)a32[k], __dmul_rn((double)lean_lds<TE>(addr + k * kstep), w));
            } else if (t.flags & TF_NEGACC) {
#pragma unroll
              for (int k = 0; k < TV; ++k) r[k] = __dsub_rn(__dmul_rn((double)lean_lds<TE>(addr + k * kstep), w), (double)a32[k]);
            } else {
#pragma unroll
              for (int k = 0; k < TV; ++k) r[k] = __dadd_rn((double)a32[k], __dmul_rn((double)lean_lds<TE>(addr + k * kstep), w));
            }
            store_bytes<double, TV>(optr, ostep, ov.dtype, cx.valid, r);
          } else if (P.n_terms > P.n32) {
            double a64[TV];
#pragma unroll
            for (int k = 0; k < TV; ++k) a64[k] = (double)a32[k];
            term_steps<TE, TV, double>(P, cx, P.n32, P.n_terms, a64);
            store_bytes<double, TV>(optr, ostep, ov.dtype, cx.valid, a64);
          } else {
            store_bytes<float, TV>(optr, ostep, ov.dtype, cx.valid, a32);
          }
        }
      } else {
        double a64[TV];
        term_steps<TE, TV, double>(P, cx, 0, P.n_terms, a64);
        store_bytes<double, TV>(optr, ostep, ov.dtype, cx.valid, a64);
      }
      optr += oplane;
    }
  }
}

// =============================================================================================
// host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_tiled_fn() {
  static const EncodeTiledFn fn = []() -> EncodeTiledFn {  // (initialised once, thread-safe)
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess) return (EncodeTiledFn)p;
    return nullptr;
  }();
  return fn;
}

static long long floor_div(long long a, long long b) {  // b > 0
  long long q = a / b;
  if ((a % b != 0) && (a < 0)) --q;
  return q;
}

bool plan_stencil_tile(const rb200_fused_op* op, int sms, bool use_terms, bool use_tma, TilePlan& T) {
  if (op->ndim != 2 && op->ndim != 3) return false;
  if (op->n_reds != 0 || op->n_axis_red_dims != 0) return false;
  if (!lean_vocabulary_only(op, false)) return false;
  const int nd = op->ndim;
  TileParams& P = T.P;
  memset(&T, 0, sizeof(T));
  P.Z = nd == 3 ? op->itershape[0] : 1;
  P.Y = op->itershape[nd - 2];
  P.X = op->itershape[nd - 1];
  if (P.X >= (1ll << 31) || P.Y >= (1ll << 31) || P.Z >= (1ll << 31)) return false;

  const ViewUse use = view_use(op);
  auto S = [&](int v, int d) -> long long {  // stride of normalised dim d (0 = z, 1 = y, 2 = x)
    if (nd == 3) return op->views[v].stride[d];
    return d == 0 ? 0 : op->views[v].stride[d - 1];
  };
  // the shift of view v from the reference view r, when v is a member of r's group: read-only, r's dtype, strides and
  // allocation, and a base offset that decomposes into a shift within +-3 planes, +-8 rows and +-8 columns
  auto group_shift = [&](int v, int r, long long* dz, long long* dy, long long* dx) -> bool {
    if (!use.read[v] || use.written[v] || op->views[v].dtype != op->views[r].dtype) return false;
    if (S(v, 0) != S(r, 0) || S(v, 1) != S(r, 1) || S(v, 2) != 1) return false;
    if (op->views[v].alloc_lo != op->views[r].alloc_lo) return false;
    const int es = op->views[r].dtype == RB200_F64 ? 8 : 4;
    const long long db = (const char*)op->views[v].base - (const char*)op->views[r].base;
    if (db % es != 0) return false;
    long long delta = db / es;
    *dz = 0;
    if (nd == 3 && S(r, 0) > 0) {
      *dz = floor_div(delta + S(r, 0) / 2, S(r, 0));
      delta -= *dz * S(r, 0);
    }
    *dy = floor_div(delta + S(r, 1) / 2, S(r, 1));
    *dx = delta - *dy * S(r, 1);
    return *dz >= -3 && *dz <= 3 && *dy >= -8 && *dy <= 8 && *dx >= -8 && *dx <= 8;
  };

  // ---- staged group: the largest family of read-only views with equal dtype and strides (unit x stride) whose base
  // offsets are small shifts of each other
  int best_ref = -1, best_n = 0;
  int member[RB200_MAX_VIEWS];
  long long mdz[RB200_MAX_VIEWS], mdy[RB200_MAX_VIEWS], mdx[RB200_MAX_VIEWS];
  for (int r = 0; r < op->n_views; ++r) {
    if (!use.read[r] || use.written[r] || S(r, 2) != 1 || S(r, 1) < 64 || (nd == 3 && S(r, 0) < S(r, 1))) continue;
    if (!op->views[r].alloc_lo || !op->views[r].alloc_hi) continue;
    int n = 0;
    long long dz, dy, dx;
    for (int v = 0; v < op->n_views; ++v)
      if (group_shift(v, r, &dz, &dy, &dx)) ++n;
    if (n > best_n) {
      best_n = n;
      best_ref = r;
    }
  }
  int view_kind[RB200_MAX_VIEWS], view_arg[RB200_MAX_VIEWS], store_arg[RB200_MAX_VIEWS];
  for (int v = 0; v < op->n_views; ++v) {
    view_kind[v] = L_DIRECT;
    view_arg[v] = 0;
    store_arg[v] = 0;
  }
  int es = 4;
  if (best_n >= 2) {
    const int r = best_ref;
    es = op->views[r].dtype == RB200_F64 ? 8 : 4;
    long long lo[3] = {0, 0, 0}, hi[3] = {0, 0, 0};
    int n = 0;
    for (int v = 0; v < op->n_views; ++v) {
      long long dz, dy, dx;
      if (!group_shift(v, r, &dz, &dy, &dx)) continue;
      member[n] = v;
      mdz[n] = dz; mdy[n] = dy; mdx[n] = dx;
      if (dz < lo[0]) lo[0] = dz;
      if (dz > hi[0]) hi[0] = dz;
      if (dy < lo[1]) lo[1] = dy;
      if (dy > hi[1]) hi[1] = dy;
      if (dx < lo[2]) lo[2] = dx;
      if (dx > hi[2]) hi[2] = dx;
      ++n;
    }
    P.has_group = 1;
    P.elem = es;
    P.hz_lo = (int)-lo[0]; P.hz = (int)(hi[0] - lo[0]);
    P.hy_lo = (int)-lo[1]; P.hy = (int)(hi[1] - lo[1]);
    P.hx_lo = (int)-lo[2]; P.hx = (int)(hi[2] - lo[2]);
    P.gs0 = S(r, 0);
    P.gs1 = S(r, 1);
    P.gcorner = (const char*)op->views[r].base - (P.hz_lo * P.gs0 + P.hy_lo * P.gs1 + P.hx_lo) * es;
    P.n_staged = n;
    // bytes any member may touch: from its first to its last element over the box
    const char* slo = nullptr;
    const char* shi = nullptr;
    for (int j = 0; j < n; ++j) {
      const char* b0 = (const char*)op->views[member[j]].base;
      const char* b1 = b0 + ((P.Z - 1) * P.gs0 + (P.Y - 1) * P.gs1 + (P.X - 1) + 1) * es;
      if (!slo || b0 < slo) slo = b0;
      if (!shi || b1 > shi) shi = b1;
    }
    P.safe_lo = slo;
    P.safe_hi = shi;
  }

  // ---- staged operands: plane of the ring and byte offset inside a plane (rows of kTilePX elements)
  if (P.has_group) {
    if (kTileTX + P.hx > kTilePX) return false;
    if (P.hz > 3) return false;
    for (int j = 0; j < P.n_staged; ++j) {
      P.staged[j].dzl = (int)(mdz[j] + P.hz_lo);
      P.staged[j].off = (unsigned)(((mdy[j] + P.hy_lo) * kTilePX + (mdx[j] + P.hx_lo)) * es);
      view_kind[member[j]] = L_STAGED;
      view_arg[member[j]] = j;
    }
  }
  // direct views: every written view, every read view outside the group
  for (int v = 0; v < op->n_views; ++v) {
    if (view_kind[v] == L_STAGED) continue;
    LDirect& d = P.direct[P.n_direct];
    d.base = (char*)op->views[v].base;
    d.s0 = S(v, 0); d.s1 = S(v, 1); d.s2 = S(v, 2);
    d.dtype = op->views[v].dtype;
    view_arg[v] = P.n_direct;
    store_arg[v] = P.n_direct;
    ++P.n_direct;
  }
  P.n_insns = op->n_insns;
  P.n_regs = op->n_regs;
  lean_translate(op, op->insns, view_kind, view_arg, store_arg, P.insns);
  P.tv = LV;
  TermBuild tb;
  tb.n_regs = P.n_regs;
  tb.direct = P.direct;
  tb.stream = false;
  tb.staged_fill = [](void* ctx, int arg, int cls_f32, TermStep* t) -> bool {
    const TileParams* Q = (const TileParams*)ctx;
    if (cls_f32 && Q->elem != 4) return false;
    if (Q->staged[arg].off > 0xffffu || Q->staged[arg].dzl > 3) return false;
    t->dzl = (unsigned char)Q->staged[arg].dzl;
    t->off = (unsigned short)Q->staged[arg].off;
    return true;
  };
  tb.ctx = &P;
  P.elem = es;
  // the term kernel runs a float32 phase only on float32 staged data (stencil_terms_kernel<float, 8>); a float64 group
  // behind a float32 prefix takes the lean machine, which runs every class
  if (!use_terms || !build_terms(tb, P.insns, P.n_insns, P.terms, kTileMaxTerms, &P.n_terms, &P.n32, &P.out_view) || (es == 8 && P.n32 > 0)) {
    P.n_terms = 0;
    P.n32 = 0;
    int n_chain = 0;
    P.n_insns = lean_fuse_chains(P.insns, P.n_insns, P.chain, kTileMaxChain, &n_chain);
  } else {
    // runs of plain `acc (+|-)= staged x` terms of one sign (the neighbour sum): the kernel walks them without decoding
    for (int i = 0; i < P.n_terms;) {
      auto plain = [&](int q) {
        const TermStep& t = P.terms[q];
        return t.kind == TK_ADD && t.xkind == X_STAGED && (t.flags & ~TF_NEGP) == 0;
      };
      if (!plain(i)) {
        ++i;
        continue;
      }
      int j = i + 1;
      while (j < P.n_terms && plain(j) && P.terms[j].flags == P.terms[i].flags && (j < P.n32) == (i < P.n32) && j - i < 250) ++j;
      P.term_run[i] = (unsigned char)(j - i);
      i = j;
    }
    if (P.n32 > 0 && P.n_terms == P.n32 + 1) {
      const TermStep& t = P.terms[P.n32];
      P.fast_tail = t.kind == TK_ADD && t.xkind == X_STAGED && (t.flags & TF_W) != 0 ? 1 : 0;
    }
  }
  for (int i = 0; i < op->n_scalars; ++i) P.scal[i] = op->scalars[i];

  // ---- tile geometry: 128 columns x (2 * tv) rows
  const int TX = kTileTX, TYr = P.tv * kTileRY;
  P.nxt = (int)((P.X + TX - 1) / TX);
  P.nyt = (int)((P.Y + TYr - 1) / TYr);
  const size_t other = (P.n_terms > 0 ? (size_t)2 * kTileMaxTerms * 4 : (size_t)P.n_regs * LV * kThreads * 8) + kTileMaxRing * 8 + 16;
  if (P.has_group) {
    P.PY = TYr + P.hy;
    if (P.PY > 256) return false;
    P.plane_bytes = (unsigned)(((size_t)kTilePX * P.PY * es + 127) / 128 * 128);
    // ring = planes in use (hz + 1) + planes in flight; two in flight when that still leaves room for two CTAs per SM
    P.prefetch = kTilePrefetch;
    while (P.prefetch > 1 && (size_t)(P.hz + 1 + P.prefetch) * P.plane_bytes + other > 100 * 1024) --P.prefetch;
    P.D = P.hz + 1 + P.prefetch;
    if (P.D > kTileMaxRing) return false;
  }
  const size_t smem = (size_t)P.D * P.plane_bytes + other;
  if (smem > 100 * 1024) return false;  // (two CTAs per SM)

  // ---- work items: z chunks so that every CTA of the persistent grid gets several
  const long long grid_cap = (long long)sms * ((P.n_terms > 0 && es == 4 && smem <= (220 * 1024) / RB200_TERMS_MINB - 1024) ? RB200_TERMS_MINB : 2);
  const long long xy = (long long)P.nxt * P.nyt;
  long long want_chunks = (grid_cap * 6 + xy - 1) / xy;
  if (want_chunks < 1) want_chunks = 1;
  long long ZC = (P.Z + want_chunks - 1) / want_chunks;
  const long long min_zc = P.has_group && P.hz > 0 ? 16 : 1;  // keep the re-read of halo planes small
  if (ZC < min_zc) ZC = min_zc;
  if (ZC > P.Z) ZC = P.Z;
  P.ZC = ZC;
  P.nzc = (int)((P.Z + ZC - 1) / ZC);
  P.n_items = (long long)P.nzc * xy;
  T.blocks = P.n_items < grid_cap ? P.n_items : grid_cap;
  T.smem = smem;
  T.es = es;
  T.nd = nd;
  // ---- can the halo'd source box be described by a TMA tensor map?  (strides multiples of 16 bytes, the corner on a
  // 16-byte boundary, rows of whole 16-byte units, the whole box inside the shard buffer.)  On an H100, bulk tensor copies
  // from maps whose base had been moved down to the boundary (shift > 0) stopped the kernel with an illegal instruction;
  // those maps' rows also ended inside a 16-byte unit and the cause is not known, so as a precaution TMA is taken only
  // where both conditions hold (DESIGN §3.4).  The shift stays in the map and kernel parameters, always 0 here.
  if (P.has_group) {
    const uintptr_t corner = (uintptr_t)P.gcorner;
    T.shift = (int)((corner & 15u) / (unsigned)es);
    T.tbase = P.gcorner - (size_t)T.shift * es;
    T.Xh = P.X + P.hx + T.shift;
    T.Yh = P.Y + P.hy;
    T.Zh = P.Z + P.hz;
    const char* far_end = P.gcorner + ((T.Zh - 1) * P.gs0 + (T.Yh - 1) * P.gs1 + (P.X + P.hx)) * es;
    const char* alo = (const char*)op->views[best_ref].alloc_lo;
    const char* ahi = (const char*)op->views[best_ref].alloc_hi;
    const bool aligned = (P.gs1 * es) % 16 == 0 && (nd == 2 || ((P.gs0 * es) % 16 == 0 && P.gs0 > 0)) && (corner % (unsigned)es) == 0;
    const bool inside = T.tbase >= alo && far_end <= ahi;
    T.tma_ok = use_tma && aligned && inside && T.shift == 0 && (T.Xh * es) % 16 == 0 && T.Xh < (1ll << 31);
  }
  return true;
}

std::string describe_stencil_tile(const TilePlan& T) {
  const TileParams& P = T.P;
  int n_chain_insns = 0, n_chain_steps = 0;
  for (int i = 0; i < P.n_insns; ++i)
    if ((P.insns[i].handler >> 2) == LO_CHAIN) {
      ++n_chain_insns;
      n_chain_steps += P.insns[i].c_arg;
    }
  char buf[400];
  snprintf(buf, sizeof(buf),
           "kernel=%s elem=%d box=%lldx%lldx%lld staged_views=%d halo=z%d+%d,y%d+%d,x%d+%d ring=%d loader=%s direct_views=%d lean_insns=%d "
           "chains=%d chain_steps=%d terms=%d(f32:%d) fast_tail=%d tile=128x%d items=%lld planes_per_item=%lld ctas=%lld smem=%zu corner_shift=%d",
           P.n_terms > 0 ? "stencil_terms" : "stencil_tile", T.es, P.Z, P.Y, P.X, P.n_staged, P.hz_lo, P.hz - P.hz_lo, P.hy_lo, P.hy - P.hy_lo, P.hx_lo, P.hx - P.hx_lo, P.D,
           !P.has_group ? "none" : (T.tma_ok ? "tma" : "cp.async"), P.n_direct, P.n_insns, n_chain_insns, n_chain_steps, P.n_terms, P.n32, P.fast_tail, P.tv * kTileRY, P.n_items,
           P.ZC, T.blocks, T.smem, P.has_group ? T.shift : 0);
  return buf;
}

cudaError_t launch_stencil_tile(TilePlan& T, cudaStream_t stream) {
  TileParams& P = T.P;
  const int es = T.es, nd = T.nd;
  CUtensorMap tmap;
  memset(&tmap, 0, sizeof(tmap));
  if (P.has_group && T.tma_ok) {
    EncodeTiledFn enc = encode_tiled_fn();
    if (enc) {
      cuuint64_t gdim[3] = {(cuuint64_t)T.Xh, (cuuint64_t)T.Yh, (cuuint64_t)T.Zh};
      cuuint64_t gstr[2] = {(cuuint64_t)(P.gs1 * es), (cuuint64_t)((nd == 3 ? P.gs0 : P.gs1 * T.Yh) * es)};
      cuuint32_t box[3] = {(cuuint32_t)kTilePX, (cuuint32_t)P.PY, 1};
      cuuint32_t estr[3] = {1, 1, 1};
      const CUresult rc = enc(&tmap, es == 8 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT64 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, (void*)T.tbase, gdim, gstr, box,
                              estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (rc == CUDA_SUCCESS) {
        P.use_tma = 1;
        P.tma_shift = T.shift;
      }
    }
  }

  static const bool attrs = []() {  // (set once, thread-safe)
    cudaFuncSetAttribute(stencil_tile_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    cudaFuncSetAttribute(stencil_tile_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    cudaFuncSetAttribute(stencil_terms_kernel<double, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    cudaFuncSetAttribute(stencil_terms_kernel<float, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    return true;
  }();
  (void)attrs;
  const unsigned blocks = (unsigned)T.blocks;
  if (P.n_terms > 0) {
    if (es == 8) stencil_terms_kernel<double, 8><<<blocks, kThreads, T.smem, stream>>>(P, tmap);
    else stencil_terms_kernel<float, 8><<<blocks, kThreads, T.smem, stream>>>(P, tmap);
  } else {
    if (es == 8) stencil_tile_kernel<double><<<blocks, kThreads, T.smem, stream>>>(P, tmap);
    else stencil_tile_kernel<float><<<blocks, kThreads, T.smem, stream>>>(P, tmap);
  }
  return cudaGetLastError();
}

}  // namespace rb200
