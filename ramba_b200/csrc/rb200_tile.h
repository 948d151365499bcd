// rb200_tile.h — parameters and host-side plan of the stencil / N-d float arithmetic kernels (rb200_tile.cu).
#pragma once
#include <cuda_runtime.h>

#include <string>

#include "rb200_lean.cuh"
#include "rb200_terms.h"

namespace rb200 {

constexpr int kTileMaxStaged = RB200_MAX_VIEWS;
constexpr int kTileMaxRing = 8;
// tile geometry (compile-time, so that every shared-memory access of an operand is base + immediate): 128 columns x
// 16 rows of outputs per plane, element k of a thread is 2 rows below element k-1; the staged box is 144 columns wide
// (halo <= 16 columns in total) and 16 + halo rows high
constexpr int kTileTX = 128, kTileLogTX = 7, kTileRY = kThreads / kTileTX, kTileTY = LV * kTileRY, kTilePX = 144;
constexpr int kTileMaxChain = 64;
constexpr int kTilePrefetch = 2;  // planes requested ahead of the one being computed (1 when the ring would not fit)

struct TileStagedOp {
  int dzl;           // plane of the ring relative to the oldest needed plane (0 .. hz)
  unsigned off;      // byte offset inside a plane: ((dy + hy_lo) * PX + dx + hx_lo) * elem
};

constexpr int kTileMaxTerms = kMaxTerms;

struct TileParams {
  long long Z, Y, X;        // iteration extents (Z == 1 for 2-D ops)
  int nxt, nyt, nzc;        // tiles along x, y; chunks along z
  long long ZC;             // planes per work item
  long long n_items;
  // staged group
  int has_group, use_tma, elem;
  int hz_lo, hz, hy_lo, hy, hx_lo, hx;  // halos: lo part and total (lo + hi)
  int PY, D, prefetch;                   // rows of the plane box (kTilePX columns), ring depth, planes requested ahead
  unsigned plane_bytes;
  const char* gcorner;                   // address of group element (z = -hz_lo, y = -hy_lo, x = -hx_lo)
  long long gs0, gs1;                    // group strides (elements) of z and y; x stride is 1
  const char* safe_lo;                   // [safe_lo, safe_hi): bytes the cooperative loader may touch
  const char* safe_hi;
  int tma_shift;                         // elements the tensor-map base was moved down (0: the planner takes TMA only for aligned corners)
  int n_staged;
  TileStagedOp staged[kTileMaxStaged];
  int n_direct;
  LDirect direct[RB200_MAX_VIEWS];
  int n_insns, n_regs;
  LInsn insns[RB200_MAX_INSNS];
  u64 scal[RB200_MAX_SCALARS];
  LChainStep chain[kTileMaxChain];
  // term form (n_terms > 0): steps [0, n32) run in float32, steps [n32, n_terms) in float64
  int n_terms, n32, out_view;
  int fast_tail;  // the float64 phase is exactly one `acc (+|-) w*x` term over a staged operand
  int tv;  // elements per thread per plane (always LV): tile rows = tv * 2
  TermStep terms[kTileMaxTerms];
  unsigned char term_run[kTileMaxTerms];  // > 0: this and the next term_run-1 terms are plain `acc (+|-)= staged x` of one sign
};

struct TilePlan {
  TileParams P;
  size_t smem;
  long long blocks;
  // TMA descriptor inputs (valid when tma_ok): base moved down to 16-byte alignment, halo'd extents
  bool tma_ok;
  const char* tbase;
  long long Xh, Yh, Zh;
  int shift, es, nd;
};

// false: the op list is not of this kernel's form.  use_terms / use_tma: the term kernel and the TMA loader may be chosen
bool plan_stencil_tile(const rb200_fused_op* op, int sms, bool use_terms, bool use_tma, TilePlan& T);
// one line for rb200_describe_plan
std::string describe_stencil_tile(const TilePlan& T);
// encodes the tensor map (the cooperative loader when that fails) and launches; sets T.P.use_tma / tma_shift
cudaError_t launch_stencil_tile(TilePlan& T, cudaStream_t stream);

}  // namespace rb200
