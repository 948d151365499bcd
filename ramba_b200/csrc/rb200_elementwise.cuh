#pragma once
// rb200_elementwise.cuh — K1-K5: fused elementwise kernel with optional global reductions,
// instantiated per iteration-space rank in rb200_elementwise_nd*.cu (parallel compilation).
#include "rb200_interp.cuh"
#include "rb200_launch.h"

namespace rb200 {

// Persistent-style grid (a multiple of the SM count): CTA b walks tiles b, b+grid, ...
// Shared memory layout (dynamic): [prefetch: 2 stages * n_pf * V*256*8 B][register file: n_regs*V*256*8 B]
// AX1D: axis reduction run as a 1-D op (ND == 1 only).  The box is [reduced rows][C kept elements] with
// C a multiple of the tile and the grid a multiple of C/TILE, so a CTA always lands on the same column
// chunk: every thread keeps V column accumulators in registers across all its rows, views that are
// broadcast over the rows are "periodic" (pf_slot == -2), and the per-CTA accumulators are written as
// partials[(split)*C + column] with split = blockIdx / (C/TILE).
// LEAN (ND == 1, rb200_elementwise_lean.cu): op lists of plain float arithmetic and sin / cos whose every instruction
// has a handler of the lean set (rb200_handlers_lean.inc), with no reductions, unmasked stores to contiguous views of
// the result's own dtype and every read view staged by bulk copies (the host checks all of it: lean_interp_eligible in
// rb200_interp_plan.cu).  The handler bodies are the full kernel's; without the generic path, the reductions and the
// converting / masked stores, ptxas keeps the whole loop in registers.
template <int V, int ND, bool AX1D = false, bool LEAN = false>
#ifndef RB200_MIN_BLOCKS
#define RB200_MIN_BLOCKS 2
#endif
__global__ void __launch_bounds__(kThreads, (ND == 1 && V <= 4) ? 3 : RB200_MIN_BLOCKS) vm_elementwise_kernel(const __grid_constant__ KParams P) {
  static_assert(!LEAN || (ND == 1 && !AX1D), "the lean kernel is the plain 1-D one");
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ __align__(8) u64 mbar_store[4];
  constexpr int TILE = kThreads * V;
  constexpr unsigned SLOT = (unsigned)(TILE * 8);  // bytes reserved per staged view per stage
  Ctx<V, ND, LEAN> cx(P);
  const unsigned smem_s = (unsigned)__cvta_generic_to_shared(smem);
  cx.tid = threadIdx.x;
  const int n_pf = (ND == 1) ? P.n_pf : 0;
  // layout: [prefetch stages 0..S-1][register file]  (stages first: 128-byte aligned)
  const unsigned pf_base = smem_s;
  const unsigned pf_stage_bytes = (unsigned)n_pf * SLOT;
  const bool bulk = (ND == 1) && n_pf > 0 && (LEAN || P.bulk);
  constexpr unsigned S = 2u;  // ring depth
  cx.regfile_s = smem_s + (n_pf > 0 ? S : 0u) * pf_stage_bytes + threadIdx.x * 8u;
  cx.ocls_s = cx.regfile_s + (unsigned)((P.n_regs + 1) * V * kThreads * 8);  // behind the register file and its scratch column  // offset-class table follows the register file
  cx.pf_s = pf_base;
  const unsigned mbar0 = (unsigned)__cvta_generic_to_shared(&mbar_store[0]);
  if (bulk) {
    if (threadIdx.x == 0) {
      for (unsigned s = 0; s < S; ++s) mbar_init(mbar0 + s * 8u, 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
  }

  // reduction accumulators: slot 0 in registers; slots 1.. (multi-reduction ops) in shared memory
  constexpr int NS = 1;
  __shared__ u64 racc_extra[RB200_MAX_REDS - 1][kThreads];
  u64 racc[NS][AX1D ? V : 1];
  if constexpr (!LEAN) {
#pragma unroll
    for (int k = 0; k < (AX1D ? V : 1); ++k) racc[0][k] = red_identity_bits(0 < P.n_reds ? P.reds[0].op : 0, 0 < P.n_reds ? P.reds[0].ctype : 0);
    cx.racc_s = (unsigned)__cvta_generic_to_shared(&racc_extra[0][threadIdx.x]);
    for (int s = 1; s < P.n_reds; ++s) racc_extra[s - 1][threadIdx.x] = red_identity_bits(P.reds[s].op, P.reds[s].ctype);
  }
  if constexpr (AX1D) {
    cx.pe0 = (long long)(blockIdx.x % (unsigned)P.n_split_chunks) * TILE + threadIdx.x;
    cx.e0 = cx.pe0;
    cx.valid = (1u << V) - 1u;
    // hoist the row-broadcast operands: this CTA always works on the same column chunk
#pragma unroll 1
    for (int h = 0; h < P.n_hoist; ++h) {
      const KView& vw = P.views[P.hoist_view[h]];
      long long off[V];
      cx.offsets(vw, off);
      u64 bits[V];
      if (P.hoist_cls[h] == RB200_T_F64) {
        double t[V];
        load_view<double, V>(vw.base, vw.dtype, off, cx.valid, t);
#pragma unroll
        for (int k = 0; k < V; ++k) bits[k] = CT<double>::bits(t[k]);
      } else if (P.hoist_cls[h] == RB200_T_F32) {
        float t[V];
        load_view<float, V>(vw.base, vw.dtype, off, cx.valid, t);
#pragma unroll
        for (int k = 0; k < V; ++k) bits[k] = CT<float>::bits(t[k]);
      } else {
        long long t[V];
        load_view<long long, V>(vw.base, vw.dtype, off, cx.valid, t);
#pragma unroll
        for (int k = 0; k < V; ++k) bits[k] = CT<long long>::bits(t[k]);
      }
      sts_vec64<V>(cx.reg_base(P.hoist_reg[h]), bits);
    }
  } else {
    cx.pe0 = 0;
  }

  // --- staging of the read-only inputs of tile t into stage `st` (ND == 1 only) --------------
  // full tiles of contiguous, 16-byte aligned views: ONE bulk async copy per view by one thread
  auto issue_bulk = [&](long long t, unsigned st) {
    const unsigned mb = mbar0 + st * 8u;
    unsigned bytes = 0;
#pragma unroll 1
    for (int j = 0; j < n_pf; ++j) {
      const int dt = P.views[P.pf_view[j]].dtype;
      bytes += (unsigned)TILE * ((dt == RB200_F64 || dt == RB200_I64) ? 8u : 4u);
    }
    mbar_expect_tx(mb, bytes);
#pragma unroll 1
    for (int j = 0; j < n_pf; ++j) {
      const KView& vw = P.views[P.pf_view[j]];
      const unsigned es = (vw.dtype == RB200_F64 || vw.dtype == RB200_I64) ? 8u : 4u;
      bulk_g2s(pf_base + st * pf_stage_bytes + (unsigned)j * SLOT, vw.base + t * (long long)TILE * es, (unsigned)TILE * es, mb);
    }
  };
  // ragged / strided / unaligned tiles: one cp.async per element, zero-filled past the end
  auto issue_ldgsts = [&](long long t, unsigned st) {
    const long long e0 = t * TILE + threadIdx.x;
    const long long left = P.total - e0;  // element k exists iff k*256 < left
#pragma unroll 1
    for (int j = 0; j < n_pf; ++j) {
      const KView& vw = P.views[P.pf_view[j]];
      const int es = (vw.dtype == RB200_F64 || vw.dtype == RB200_I64) ? 8 : 4;
      const long long sb = vw.stride[0] * es;  // byte stride per element (uniform)
      const long long step = sb * kThreads;
      const char* src = vw.base + e0 * sb;
      unsigned dst = pf_base + st * pf_stage_bytes + (unsigned)j * SLOT + threadIdx.x * (unsigned)es;
#pragma unroll
      for (int k = 0; k < V; ++k) {
        const bool ok = (long long)k * kThreads < left;
        if (es == 8) cp_async8(dst, ok ? src : vw.base, ok);
        else cp_async4(dst, ok ? src : vw.base, ok);
        src += step;
        dst += (unsigned)(kThreads * es);
      }
    }
  };
  auto tile_is_bulk = [&](long long t) { return bulk && (t + 1) * TILE <= P.total; };

  // Ring protocol (bulk mode).  Stage s = it mod S holds the CTA's it-th tile (S a power of two); its
  // "full" mbarrier completes once per refill, so the it-th tile waits for parity (it / S) & 1.  One
  // CTA-wide barrier per tile guards the refill of the stage the previous tile used.  (A barrier-free
  // variant -- warps count themselves out of a stage, the last one out refills it -- measured 8 % slower
  // on config 2: the barrier keeps the eight warps in step, which the instruction cache likes.)
  constexpr unsigned lgS = 1u;
  if (n_pf > 0 && (long long)blockIdx.x < P.n_tiles) {
    if (bulk) {
      if (threadIdx.x == 0) {
        long long t = blockIdx.x;
        for (unsigned s = 0; s < S && t < P.n_tiles; ++s, t += gridDim.x)
          if (tile_is_bulk(t)) issue_bulk(t, s);
      }
    } else {
      issue_ldgsts(blockIdx.x, 0);
      cp_async_commit();
    }
  }
#pragma unroll 1
  for (unsigned it = 0;; ++it) {
    // per-tile quantities are re-derived from the tile counter and constant-bank values (kept opaque so
    // that they are not hoisted into registers that stay live across the whole interpreter)
    unsigned grid = gridDim.x;
    asm volatile("" : "+r"(grid));
    const long long tile = (long long)blockIdx.x + (long long)it * grid;
    if (tile >= P.n_tiles) break;
    const unsigned stage = bulk ? (it & (S - 1u)) : (it & 1u);
    if (n_pf > 0) {
      if (bulk) {
        // everybody is done reading the stage used by the previous iteration before it is refilled
        __syncthreads();
        if (it > 0 && threadIdx.x == 0) {
          const long long nxt = tile + (long long)(S - 1u) * grid;
          if (nxt < P.n_tiles && tile_is_bulk(nxt)) issue_bulk(nxt, (it - 1u) & (S - 1u));
        }
        if (tile_is_bulk(tile)) {
          mbar_wait(mbar0 + stage * 8u, (it >> lgS) & 1u);
        } else {  // the ragged last tile: every thread copies (and later reads) only its own column
          issue_ldgsts(tile, stage);
          cp_async_commit();
          cp_async_wait<0>();
        }
      } else {
        // per-thread pipeline (each thread re-reads only what it copied itself: no barrier)
        const long long nxt = tile + grid;
        if (nxt < P.n_tiles) issue_ldgsts(nxt, stage ^ 1u);
        cp_async_commit();
        cp_async_wait<1>();
      }
      cx.pf_s = pf_base + stage * pf_stage_bytes;
    }
    const long long e0 = tile * TILE + threadIdx.x;
    unsigned valid = 0;
    if constexpr (ND == 1) {
      cx.e0 = e0;
      if ((tile + 1) * TILE <= P.total) {  // full tile (uniform): no per-element bounds checks
        valid = (1u << V) - 1u;
      } else {
#pragma unroll
        for (int k = 0; k < V; ++k)
          if (e0 + (long long)k * kThreads < P.total) valid |= (1u << k);
      }
    } else if (P.row_chunks > 0) {
      // row mode: this tile is chunk `ch` of row `row` of the innermost dim; outer indices are per tile
      long long row, ch;
      if (((tile | (long long)P.row_chunks) >> 31) == 0) row = (long long)((unsigned)tile / (unsigned)P.row_chunks);
      else row = tile / P.row_chunks;
      ch = tile - row * P.row_chunks;
      long long oidx[ND];
#pragma unroll
      for (int d = ND - 1; d >= 0; --d) {
        if (d >= P.ndim - 1) {
          oidx[d] = 0;
        } else if (d == 0) {
          oidx[d] = row;
        } else {
          const long long sd = P.shape[d];
          long long q;
          if (((row | sd) >> 31) == 0) q = (long long)((unsigned)row / (unsigned)sd);
          else q = row / sd;
          oidx[d] = row - q * sd;
          row = q;
        }
      }
      const long long inner = P.shape[P.ndim - 1];
      const long long j0 = ch * TILE + threadIdx.x;
#pragma unroll
      for (int k = 0; k < V; ++k) {
        const long long j = j0 + (long long)k * kThreads;
        const bool ok = j < inner;
        if (ok) valid |= (1u << k);
#pragma unroll
        for (int d = 0; d < ND; ++d) cx.idx[k][d] = (d == P.ndim - 1) ? (ok ? j : 0) : (ok ? oidx[d] : 0);
      }
    } else {
#pragma unroll
      for (int k = 0; k < V; ++k) {
        const long long e = e0 + (long long)k * kThreads;
        if (e < P.total) {
          valid |= (1u << k);
          decode_index<ND>(P, e, 0, cx.idx[k]);
        } else {
#pragma unroll
          for (int d = 0; d < ND; ++d) cx.idx[k][d] = 0;
        }
      }
    }
    cx.valid = valid;
    cx.fill_offset_classes();
    run_program<V, AX1D, NS, LEAN>(cx, racc);
  }
  if constexpr (LEAN) return;
  if (n_pf > 0 && !bulk) cp_async_wait<0>();

  if constexpr (AX1D) {
    // per-CTA column accumulators -> partials[split][column]
    const long long split = blockIdx.x / (unsigned)P.n_split_chunks;
    const long long col0 = cx.pe0;
#pragma unroll
    for (int k = 0; k < V; ++k) P.red_partials[split * P.red_len + col0 + (long long)k * kThreads] = racc[0][k];
    return;
  }
  // ---- global reductions: thread -> warp shuffle -> block -> per-block partial -> last block
  if (P.n_reds > 0) {
    __shared__ u64 wpart[RB200_MAX_REDS][kThreads / 32];
    __shared__ bool is_last;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int s = 0; s < P.n_reds; ++s) {
      const int op = P.reds[s].op, ct = P.reds[s].ctype;
      u64 v = (s == 0) ? racc[0][0] : racc_extra[s > 0 ? s - 1 : 0][threadIdx.x];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v = red_combine_bits(op, ct, v, __shfl_down_sync(0xffffffffu, v, o));
      if (lane == 0) wpart[s][warp] = v;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int s = 0; s < P.n_reds; ++s) {
        const int op = P.reds[s].op, ct = P.reds[s].ctype;
        u64 v = wpart[s][0];
        for (int q = 1; q < kThreads / 32; ++q) v = red_combine_bits(op, ct, v, wpart[s][q]);
        P.red_partials[(long long)s * gridDim.x + blockIdx.x] = v;
      }
      __threadfence();
      unsigned prev = atomicAdd(P.red_counter, 1u);
      is_last = (prev == gridDim.x - 1);
    }
    __syncthreads();
    if (is_last) {
      __threadfence();
      for (int s = 0; s < P.n_reds; ++s) {
        const int op = P.reds[s].op, ct = P.reds[s].ctype;
        // fixed order: thread t folds partials t, t+256, ...; then the same tree as above
        u64 v = red_identity_bits(op, ct);
        for (unsigned b = threadIdx.x; b < gridDim.x; b += kThreads) v = red_combine_bits(op, ct, v, __ldcg(&P.red_partials[(long long)s * gridDim.x + b]));
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v = red_combine_bits(op, ct, v, __shfl_down_sync(0xffffffffu, v, o));
        __syncthreads();
        if (lane == 0) wpart[s][warp] = v;
        __syncthreads();
        if (threadIdx.x == 0) {
          v = wpart[s][0];
          for (int q = 1; q < kThreads / 32; ++q) v = red_combine_bits(op, ct, v, wpart[s][q]);
          // red[0,..] = red[0,..] (op) acc  (ramba/ramba.py:5805-5806), rounded to the partial
          // array's dtype on store
          void* out = P.reds[s].out;
          const double vd = (ct == RB200_T_F64) ? CT<double>::get(v) : (double)(long long)v;
          const long long vi = (ct == RB200_T_F64) ? (long long)CT<double>::get(v) : (long long)v;
          switch (P.reds[s].out_dtype) {
            case RB200_F64: { double* o = (double*)out; *o = red_combine<double>(op, *o, vd); } break;
            case RB200_F32: { float* o = (float*)out; *o = (float)red_combine<double>(op, (double)*o, vd); } break;
            case RB200_I64: { long long* o = (long long*)out; *o = red_combine<long long>(op, *o, vi); } break;
            case RB200_I32: { int* o = (int*)out; *o = (int)red_combine<long long>(op, (long long)*o, vi); } break;
            case RB200_BOOL: { unsigned char* o = (unsigned char*)out; *o = red_combine<long long>(op, (long long)*o, vi) != 0 ? 1 : 0; } break;
            case RB200_U8: { unsigned char* o = (unsigned char*)out; *o = (unsigned char)red_combine<long long>(op, (long long)*o, vi); } break;
            case RB200_I8: { signed char* o = (signed char*)out; *o = (signed char)red_combine<long long>(op, (long long)*o, vi); } break;
            case RB200_I16: { short* o = (short*)out; *o = (short)red_combine<long long>(op, (long long)*o, vi); } break;
            case RB200_U16: { unsigned short* o = (unsigned short*)out; *o = (unsigned short)red_combine<long long>(op, (long long)*o, vi); } break;
            case RB200_U32: { unsigned int* o = (unsigned int*)out; *o = (unsigned int)red_combine<long long>(op, (long long)*o, vi); } break;
            default: break;
          }
        }
      }
      if (threadIdx.x == 0) *P.red_counter = 0u;  // leave scratch ready for the next launch
    }
  }
}

template <int V, int ND, bool AX1D = false, bool LEAN = false>
cudaError_t launch_vm_elementwise_nd(const KParams& P, unsigned blocks, size_t smem, cudaStream_t stream) {
  if (smem + 2048 > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(vm_elementwise_kernel<V, ND, AX1D, LEAN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  vm_elementwise_kernel<V, ND, AX1D, LEAN><<<blocks, kThreads, smem, stream>>>(P);
  return cudaGetLastError();
}

}  // namespace rb200
