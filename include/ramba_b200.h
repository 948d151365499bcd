/*
 * ramba_b200.h — C-ABI of libramba_b200.so (sm_90a), the execution seam of the
 * fused elementwise / reduction / shifted-slice hot path.
 *
 * What it replaces in the reference (Python-for-HPC/ramba, all file:line relative to
 * the reference tree):
 *
 *   rb200_run_deferred_ops   <- RemoteState.run_deferred_ops kernel launch,
 *                               ramba/ramba.py:3758-3780: one call runs one fused
 *                               op over ONE iteration range of ONE worker, with the
 *                               generated-kernel signature
 *                               f(global_start, itershape, worker_num, num_workers,
 *                                 *array_views, *scalars)   (ramba/ramba.py:8262, 8265).
 *                               The Python-source kernel body (ramba/ramba.py:8247-8255)
 *                               becomes the op-list `insns`; the per-view NumPy views
 *                               (shardview.array_to_view, ramba/shardview_array.py:557-614)
 *                               become `rb200_view` stride descriptors; pickled scalars
 *                               (ramba/ramba.py:3661-3666) become `scalars`; pre/postcode
 *                               of global reductions (ramba/ramba.py:5798-5807) and the
 *                               axis-reduction loop nest (ramba/ramba.py:8231-8244)
 *                               become the `red_*` fields.
 *   rb200_reduce_partials    <- stage 2 of an axis reduction over partial slices,
 *                               ndarray.internal_reduction2_executor, ramba/ramba.py:5818-5849.
 *   rb200_cumulative         <- RemoteState.scumulative_worker, ramba/ramba.py:3378-3437 (cumsum / scumulative).
 *   rb200_last_error         <- worker exception -> ("ERROR", worker, traceback) reply,
 *                               ramba/ramba.py:3875-3881.
 *
 * Ownership: every device pointer is BORROWED for the duration of one call (the
 * Python side owns shards as torch tensors keyed by gid, like the worker's
 * numpy_map, ramba/ramba.py:1898, 2005). Launches are asynchronous on `stream`.
 * All entry points return 0 on success, non-zero on error (see rb200_last_error).
 * There is no CPU fallback: without a CUDA device every launch fails.
 */
#ifndef RAMBA_B200_H
#define RAMBA_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RB200_ABI_VERSION 7

#define RB200_MAX_DIMS 5     /* iteration dims after host-side collapsing            */
#define RB200_MAX_VIEWS 16   /* distinct array views per fused op                    */
#define RB200_MAX_SCALARS 32 /* scalar table entries                                 */
#define RB200_MAX_INSNS 96   /* op-list length                                       */
#define RB200_MAX_REGS 12    /* spill registers of the accumulator machine           */
#define RB200_MAX_REDS 4     /* global reductions fused into one op                  */

/* storage dtypes of array views */
enum rb200_dtype {
  RB200_F64 = 0,
  RB200_F32 = 1,
  RB200_I64 = 2,
  RB200_I32 = 3,
  RB200_BOOL = 4, /* 1 byte, 0/1 */
  RB200_U8 = 5,
  RB200_I8 = 6,
  RB200_I16 = 7,
  RB200_U16 = 8,
  RB200_U32 = 9,
  RB200_NUM_DTYPES = 10
};

/* compute classes of the op-list machine (what Numba's scalar typing gives the
 * reference's generated loop body) */
enum rb200_ctype { RB200_T_F64 = 0, RB200_T_F32 = 1, RB200_T_I64 = 2 };

/* operand kinds */
enum rb200_kind {
  RB200_K_NONE = 0,
  RB200_K_ACC = 1,  /* result of the previous instruction                           */
  RB200_K_REG = 2,  /* spill register idx                                           */
  RB200_K_VIEW = 3, /* element of views[idx] at the current index                   */
  RB200_K_SCAL = 4, /* scalars[idx] (already in the instruction's compute class)    */
  RB200_K_IOTA = 5  /* index[idx] + global_start[idx]  (ramba/ramba.py:8955-8960)   */
};

/* opcodes; vocabulary = the reference's op tables, ramba/ramba.py:7893-7993 */
enum rb200_op {
  RB200_OP_MOV = 0,
  RB200_OP_ADD = 1,
  RB200_OP_SUB = 2,
  RB200_OP_MUL = 3,
  RB200_OP_DIV = 4,      /* true division                                         */
  RB200_OP_FLOORDIV = 5, /* Python semantics                                      */
  RB200_OP_MOD = 6,      /* Python semantics                                      */
  RB200_OP_POW = 7,      /* float ** float                                        */
  RB200_OP_POWI = 8,     /* x ** int64 by repeated squaring (Numba int_power)     */
  RB200_OP_MIN = 9,      /* builtins.min(a,b)                                     */
  RB200_OP_MAX = 10,     /* builtins.max(a,b)                                     */
  RB200_OP_GT = 11,
  RB200_OP_LT = 12,
  RB200_OP_GE = 13,
  RB200_OP_LE = 14,
  RB200_OP_EQ = 15,
  RB200_OP_NE = 16,
  RB200_OP_LAND = 17,
  RB200_OP_LOR = 18,
  RB200_OP_LXOR = 19,
  RB200_OP_BAND = 20,
  RB200_OP_BOR = 21,
  RB200_OP_BXOR = 22,
  RB200_OP_SHL = 23,
  RB200_OP_SHR = 24,
  RB200_OP_ABS = 25,
  RB200_OP_SQUARE = 26,
  RB200_OP_SQRT = 27,
  RB200_OP_SIN = 28,
  RB200_OP_COS = 29,
  RB200_OP_TAN = 30,
  RB200_OP_SINH = 31,
  RB200_OP_COSH = 32,
  RB200_OP_TANH = 33,
  RB200_OP_ASIN = 34,
  RB200_OP_ACOS = 35,
  RB200_OP_ATAN = 36,
  RB200_OP_NEG = 37,
  RB200_OP_EXP = 38,
  RB200_OP_LOG = 39,
  RB200_OP_ISFINITE = 40,
  RB200_OP_ISINF = 41,
  RB200_OP_ISNAN = 42,
  RB200_OP_ISNEGINF = 43,
  RB200_OP_ISPOSINF = 44,
  RB200_OP_LNOT = 45,
  RB200_OP_INVERT = 46,
  RB200_OP_WHERE = 47,  /* a ? b : c  (a is tested != 0 in the compute class)      */
  RB200_OP_CVT = 48,    /* convert a from class `imm & 0xff` to `ctype`; if
                           (imm >> 8) != 0 first wrap/round through storage dtype
                           ((imm >> 8) - 1), i.e. the value a store + reload yields */
  RB200_OP_SINCOS = 49, /* acc = sin(a), regs[st2] = cos(a) (imm 1: swapped); one range
                           reduction for both.  If c_kind == RB200_K_VIEW the parked
                           half is also stored to views[c_idx]                       */
  RB200_OP_RED = 50,    /* red[b_idx] = red[b_idx] (+,*,min,max by imm) a          */
  RB200_OP_CBRT = 51,
  /* three-operand forms of `a (+/-) b*c`: the product and the sum are rounded SEPARATELY (no FMA), exactly like the
     two statements of the reference's loop body they stand for; they exist so that a weighted term of a stencil
     (`... - 6.0*U[...]`, ramba/ramba.py:8146-8188) does not need a spill register                                */
  RB200_OP_MULADD = 52,  /* a + b*c                                                */
  RB200_OP_MULSUB = 53,  /* a - b*c                                                */
  RB200_OP_MULRSUB = 54, /* b*c - a                                                */
  RB200_OP_PHILOX = 55,  /* counter-based random draw: element value = f(a, key); see below      */
  RB200_NUM_OPS = 56
};

/* RB200_OP_PHILOX: one element of a random draw, a pure function of (key, index), so that the values do not depend on
 * how the array is partitioned, on the number of ranks or on what the draw is fused with.
 *   a: the int64 global C-order linear index i of the element in the drawn array (IOTA, ACC or REG)
 *   b: RB200_K_SCAL, the 64-bit key of the draw (the Python layer derives it as
 *        key = splitmix64(splitmix64(seed) ^ draw_number)
 *      where draw_number counts the draws made from one generator state since it was seeded)
 *   c: RB200_K_SCAL, the bound n >= 1 of the integer form (ignored by the other forms)
 *   imm: the output form (rb200_philox_form); ctype must be the form's class.
 * Block: philox4x32_10(counter, key) is Philox4x32-10 (Salmon et al., SC'11, "Random123") with
 *   key = (key_lo32, key_hi32) and counter = (j_lo32, j_hi32, 0, 0), giving words w0..w3; half h of the block is the
 *   64-bit integer x_h = w_{2h} | w_{2h+1} << 32.  Counter 0, key 0 gives 6627e8d5 e169c58d bc57ac4c 9b00dbd8.
 * Forms (j = the block element i reads):
 *   UNIFORM64 (F64): j = i >> 1, x = x_{i & 1}, value (x >> 11) * 2^-53, in [0, 1)
 *   UNIFORM32 (F32): j = i >> 2, w = w_{i & 3}, value (w >> 8) * 2^-24, in [0, 1)
 *   NORMAL64  (F64): j = i >> 1, Box-Muller with every step rounded separately: u1 = 1 - (x_0 >> 11) * 2^-53 in (0, 1],
 *                    u2 = (x_1 >> 11) * 2^-53, r = sqrt(-2 * log(u1)), t = 2*pi * u2; element 2j is r*cos(t), 2j+1 is
 *                    r*sin(t).  log, sqrt, sin and cos are the CUDA double-precision functions (not bit-identical
 *                    to a host libm: the last bits may differ)
 *   INTEGER   (I64): j = i >> 1, x = x_{i & 1}, value mulhi64(x, n) in [0, n); P(v) differs from 1/n by at most
 *                    1/2^64 (the bias of a multiply-shift reduction is below n / 2^64 overall)                          */
enum rb200_philox_form {
  RB200_PHILOX_UNIFORM64 = 0,
  RB200_PHILOX_UNIFORM32 = 1,
  RB200_PHILOX_NORMAL64 = 2,
  RB200_PHILOX_INTEGER = 3
};

enum rb200_redop { RB200_RED_ADD = 0, RB200_RED_MUL = 1, RB200_RED_MIN = 2, RB200_RED_MAX = 3 };

#define RB200_NOSTORE 0xff

/* one op-list instruction, 16 bytes */
typedef struct rb200_insn {
  uint8_t op;      /* rb200_op                                                     */
  uint8_t ctype;   /* compute class operands are fetched in / op is evaluated in   */
  uint8_t a_kind, a_idx;
  uint8_t b_kind, b_idx;
  uint8_t c_kind, c_idx;
  uint8_t st_reg;  /* also copy the result into spill register (RB200_NOSTORE: no) */
  uint8_t st_view; /* also store the result into views[st_view] (converted to its
                      dtype)                                                       */
  uint8_t st2;     /* second result register (SINCOS)                              */
  uint8_t mask_reg;/* RB200_NOSTORE, or spill register holding the write mask of a
                      masked store  (`if mask[index]:` guard, ramba/ramba.py:8476) */
  uint32_t imm;
} rb200_insn;

/* one array view bound to one iteration range: element (i0..ik) of the range lives
 * at base + sum(i_d * stride[d]) elements.  stride 0 = broadcast axis
 * (axis_map == -1, ramba/shardview_array.py:36).                                  */
typedef struct rb200_view {
  void* base;
  int64_t stride[RB200_MAX_DIMS];
  int32_t dtype; /* rb200_dtype */
  int32_t flags; /* bit0: written by this op                                       */
  /* [alloc_lo, alloc_hi): the device buffer `base` points into (the worker's shard, LocalNdarray.bcontainer,
   * ramba/ramba.py:1208-1214).  Optional (both NULL = unknown).  The stencil kernel stages a tile plus its halo
   * with whole-box TMA copies only when the box lies inside these bounds.                                       */
  const void* alloc_lo;
  const void* alloc_hi;
} rb200_view;

typedef struct rb200_red {
  int32_t op;    /* rb200_redop                                                    */
  int32_t ctype; /* accumulator class: RB200_T_F64 or RB200_T_I64                  */
  void* out;     /* device pointer to this worker's element of the partial array
                    (red[0,..] = red[0,..] (op) acc, ramba/ramba.py:5805-5806)       */
  int32_t out_dtype;
  int32_t pad;
} rb200_red;

/* One fused op over one iteration range of one worker. */
typedef struct rb200_fused_op {
  int32_t abi_version; /* RB200_ABI_VERSION                                        */
  int32_t ndim;        /* 1..RB200_MAX_DIMS (collapsed iteration space)            */
  int64_t itershape[RB200_MAX_DIMS];
  int64_t global_start[RB200_MAX_DIMS]; /* added to IOTA operands                   */
  int32_t iota_dim[RB200_MAX_DIMS];     /* unused (reserved)                        */
  int32_t worker_num, num_workers;
  int32_t n_views, n_scalars, n_insns, n_regs, n_reds;
  /* axis reduction (ramba/ramba.py:8231-8244): the host orders the iteration dims
   * [reduced..., kept...]; the first n_axis_red_dims dims are walked sequentially per
   * output element (split into axis_nsplit slices for parallelism) and every RED slot
   * s leaves raw 64-bit partials of its accumulator class in
   *   red_scratch[(s*axis_nsplit + split)*kept_elems + kept_linear_index].
   * 0 = not an axis reduction (RED slots are global reductions written to reds[].out). */
  int32_t n_axis_red_dims;
  int32_t axis_nsplit;
  rb200_view views[RB200_MAX_VIEWS];
  uint64_t scalars[RB200_MAX_SCALARS]; /* raw bits: double / float(low 32) / int64 */
  rb200_insn insns[RB200_MAX_INSNS];
  rb200_red reds[RB200_MAX_REDS];
  /* scratch for cross-block reduction: >= rb200_red_scratch_bytes() bytes, zeroed
   * once at allocation (the kernel leaves its counters zero on exit)               */
  void* red_scratch;
} rb200_fused_op;

/* Launch one fused op on `stream` (a cudaStream_t, may be NULL = legacy default).   */
int rb200_run_deferred_ops(const rb200_fused_op* op, void* stream);

/* Bytes of zero-initialised device scratch a launch with reductions needs.          */
int64_t rb200_red_scratch_bytes(void);

/* out[j] = reduce_k partial[k*stride_k + j], j < n  (stage 2 of an axis reduction). */
int rb200_reduce_partials(void* out, const void* partials, int64_t n, int64_t k, int64_t stride_k,
                          int32_t dtype, int32_t redop, void* stream);

/* Inclusive cumulative scan (cumsum / scumulative with +, *, min, max) of one worker's block, replacing
 * RemoteState.scumulative_worker (ramba/ramba.py:3378-3437): the block is [n_outer][len][n_inner] elements in C order,
 * the scan runs along `len`.  dtype: RB200_F64 / F32 (float64 accumulation) or RB200_I64 / I32 (int64 accumulation).
 * carry_in (optional): one accumulator-class value per sequence (n_outer * n_inner), the total of the blocks that
 * precede this one along the axis; totals_out (optional): each sequence's inclusive total.  `scratch` must hold
 * rb200_cumulative_scratch_bytes() bytes.  src == dst is allowed.  One read and one write of every element.         */
int64_t rb200_cumulative_scratch_bytes(int64_t n_outer, int64_t len, int64_t n_inner);
int rb200_cumulative(const void* src, void* dst, int32_t dtype, int64_t n_outer, int64_t len, int64_t n_inner,
                     int32_t redop, const void* carry_in, void* totals_out, void* scratch, void* stream);

/* ---- integer-array indexing (a[idx], a[idx] = v): data movement at computed addresses ----------------------------------
 * What it stands for in the reference: getitem_array_executor / setitem_array_executor (ramba/ramba.py:6429-6545,
 * 6143-6297), which move one element at a time in Python.  The host computes `lin`, the C-order linear index of every
 * addressed element within the view (int64, -1 for an element with an out-of-range coordinate); these entry points move
 * the elements.  Semantics shared by all three:
 *   - an entry of lin outside [0, view size) is added to *bad (a device uint64 counter, may be NULL when n == 0) and is
 *     never read or written;
 *   - everything is enqueued on `stream`, and nothing synchronises with the host;
 *   - malformed arguments (elem_bytes not 1/2/4/8, ndim out of range, a null pointer with n > 0, a view outside its
 *     [alloc_lo, alloc_hi), a route table that is not a grid or has too many ranks) are rejected with a reason through
 *     rb200_last_error before any device query.                                                                        */
#define RB200_MAX_ROUTE_RANKS 64  /* owners of a route table                                  */
#define RB200_MAX_ROUTE_CELLS 64  /* cells of a route table (the product of the cells per dim)  */
#define RB200_MAX_ROUTE_CUTS 40   /* cut points of a route table, all dims together            */

/* An N-d view addressed by the C-order linear index of its elements: element (c0..c_{k-1}) lives at
 * base + elem_bytes * sum(c_d * stride[d]).  Strides are in elements and may be negative or 0; a padded shard is a view
 * with the padded block's strides.  [alloc_lo, alloc_hi) is the allocation the view lies in; when both are non-NULL the
 * library checks the view's first and last reachable bytes against it.                                                  */
typedef struct rb200_index_view {
  void* base;
  int32_t ndim;       /* 1..RB200_MAX_DIMS                                        */
  int32_t elem_bytes; /* 1, 2, 4 or 8                                             */
  int64_t shape[RB200_MAX_DIMS];
  int64_t stride[RB200_MAX_DIMS];
  const void* alloc_lo;
  const void* alloc_hi;
} rb200_index_view;

/* out[i] = view[lin[i]], i < n (out is contiguous, elem_bytes per element).                                            */
int rb200_gather(const rb200_index_view* view, const int64_t* lin, int64_t n, void* out, uint64_t* bad, void* stream);

/* view[lin[i]] = values[i], i < n (values contiguous).  With duplicate entries in lin one of the values lands.         */
int rb200_scatter(const rb200_index_view* view, const int64_t* lin, int64_t n, const void* values, uint64_t* bad, void* stream);

/* The partition of a distributed view as a grid (host memory, read during the call).  Along dim d the view is cut at
 * cuts[cut_start[d] .. cut_start[d] + n_cells[d]] (ascending, 0 first, shape[d] last); cell (j0..j_{k-1}) (C order over
 * the cell grid) is held by rank cell_owner[cell], whose element (c0..) of the view lies at local element offset
 * cell_offset[cell] + sum((c_d - cuts[cut_start[d] + j_d]) * cell_stride[cell * ndim + d]) of its shard.           */
typedef struct rb200_route_table {
  int32_t ndim;
  int32_t n_ranks; /* 1..RB200_MAX_ROUTE_RANKS                                 */
  int64_t shape[RB200_MAX_DIMS];
  int32_t n_cells[RB200_MAX_DIMS];
  int32_t cut_start[RB200_MAX_DIMS];
  const int64_t* cuts;
  const int32_t* cell_owner;
  const int64_t* cell_offset;
  const int64_t* cell_stride;
} rb200_route_table;

/* Route the requests lin[0..n) to the ranks that own them.  counts[r] (n_ranks entries) receives the number of valid
 * requests owned by rank r; the requests are grouped by owner, rank 0's first, in the order of i inside each group, so the
 * grouping is a pure function of the input: slots[i] is request i's position in that grouping (-1 for an out-of-range
 * entry) and offsets[slots[i]] its owner's local element offset.  `scratch` holds rb200_route_scratch_bytes(n, n_ranks)
 * bytes.                                                                                                              */
int64_t rb200_route_scratch_bytes(int64_t n, int32_t n_ranks);
int rb200_route(const rb200_route_table* table, const int64_t* lin, int64_t n, int64_t* offsets, int64_t* slots, int64_t* counts,
                uint64_t* bad, void* scratch, void* stream);

/* ---- grouped reduction along one axis (groupby) -----------------------------------------------------------------------
 * What it stands for in the reference: RambaGroupby's aggregations (ramba/ramba.py:10185-10643), sreduce_index over Python
 * callables.  The host turns the labels of the grouped axis into a CSR table once; one launch reads every source element
 * once and writes every output once.
 *   SUM, PROD, MIN, MAX: as the engine's reductions (MIN / MAX: `b < a ? b : a`, so a NaN member is skipped);
 *   NANSUM: the sum of the members that are not NaN; NANCOUNT: their number;
 *   SQDEV: sum((x - center[o, g, i])**2), the difference and the square rounded separately.
 * Accumulator class of `out`: F64 for float sources and for SQDEV, I64 (wrapping) for integer sources otherwise.  An empty
 * group gets the identity: 0, 1, the largest / smallest value of the class (+-inf for F64), 0, 0, 0.
 * Fold order: the axis is cut into chunks of C consecutive positions (rb200_describe_group_plan states C, a function of the
 * view's shape and G only); the members of a group inside a chunk are combined in ascending order starting from the
 * identity, and the chunk partials in chunk order, again starting from the identity.  No atomics.                     */
enum rb200_group_op {
  RB200_GROUP_SUM = 0,
  RB200_GROUP_PROD = 1,
  RB200_GROUP_MIN = 2,
  RB200_GROUP_MAX = 3,
  RB200_GROUP_NANSUM = 4,
  RB200_GROUP_NANCOUNT = 5,
  RB200_GROUP_SQDEV = 6,
  RB200_GROUP_NUM_OPS = 7
};

typedef struct rb200_group_table {
  int32_t n_groups;        /* G >= 1                                                                              */
  int64_t len;             /* extent of the grouped axis in this view                                             */
  const int64_t* offsets;  /* device, G+1 entries: offsets[0] = 0, ascending, offsets[G] = len                    */
  const int64_t* members;  /* device, len entries: positions along the axis, grouped by label and ascending inside
                              each group (a permutation of 0..len-1)                                              */
} rb200_group_table;

/* out[o, g, i] = op over t in members[offsets[g]:offsets[g+1]] of src[o, t, i] (o: the axes before `axis`, i: the axes
 * after it).  src_dtype: RB200_F64, F32, I64 or I32 (matching src->elem_bytes).  out is contiguous in the accumulator
 * class; center (SQDEV only): the same shape as out, F64.  scratch: rb200_group_reduce_scratch_bytes() bytes (may be NULL
 * when that is 0).  Malformed arguments are rejected with a reason before any device query.                          */
int rb200_group_reduce(const rb200_index_view* src, int32_t src_dtype, int32_t axis, const rb200_group_table* groups, int32_t op,
                       const void* center, void* out, void* scratch, void* stream);
int64_t rb200_group_reduce_scratch_bytes(const rb200_index_view* src, int32_t axis, int32_t n_groups);
/* One text line: form (row / column / general), chunk C, chunks, CTAs, scratch.  Needs no device.  NULL on a malformed
 * argument (reason in rb200_last_error); the text stays valid until the next call on this thread.                    */
const char* rb200_describe_group_plan(const rb200_index_view* src, int32_t axis, int32_t n_groups);

/* ---- first-occurrence index reductions (argmax, argmin, nanargmax, nanargmin) ------------------------------------------
 * Every element of the view becomes an int64 order key:
 *   - an integer: its value;
 *   - a float: -0.0 becomes +0.0, then its bit pattern b (float32: the 32-bit pattern, sign-extended) gives
 *     b >= 0 ? b : b ^ INT64_MAX; a NaN gives INT64_MAX for ARG_MAX and INT64_MIN for ARG_MIN;
 *   - ARG_MIN and ARG_NANMIN then take ~key;
 *   - ARG_NANMAX and ARG_NANMIN give a NaN element no candidate.
 * Every op is then "the largest key, then the smallest index", a total order, so the result does not depend on the
 * launch shape.  An output with no candidate (an empty extent, or only NaN in a nan variant) gets index INT64_MAX and
 * key INT64_MIN.
 * Indices are global: the caller gives origin[d], the global coordinate of the view's element (0, ..., 0), and
 * gstride[d], the C-order strides of the global array's shape (host arrays of src->ndim entries, read during the call).
 *   axis = RB200_ARG_ALL_AXES: one output, the flat C-order index sum((origin[d] + c_d) * gstride[d]);
 *   axis = k: one output per kept element (C order over the view's dims without k), the position origin[k] + c_k.
 * out_idx and out_key: device, one int64 per output.  src_dtype: RB200_F64, F32, I64 or I32 (matching
 * src->elem_bytes).  scratch: rb200_arg_reduce_scratch_bytes() bytes (may be NULL when that is 0).  Malformed arguments
 * are rejected with a reason before any device query.                                                                */
enum rb200_arg_op { RB200_ARG_MAX = 0, RB200_ARG_MIN = 1, RB200_ARG_NANMAX = 2, RB200_ARG_NANMIN = 3, RB200_ARG_NUM_OPS = 4 };
#define RB200_ARG_ALL_AXES (-1)

int rb200_arg_reduce(const rb200_index_view* src, int32_t src_dtype, int32_t axis, int32_t op, const int64_t* origin, const int64_t* gstride,
                     int64_t* out_idx, int64_t* out_key, void* scratch, void* stream);
int64_t rb200_arg_reduce_scratch_bytes(const rb200_index_view* src, int32_t axis);
/* One text line: form (global / row / column / general), chunk, split, outputs, CTAs, scratch.  Needs no device.  NULL
 * on a malformed argument (reason in rb200_last_error); the text stays valid until the next call on this thread.      */
const char* rb200_describe_arg_plan(const rb200_index_view* src, int32_t axis);

/* ---- stream compaction (nonzero, flatnonzero, extract) ---------------------------------------------------------------
 * An element of the condition view is selected when its stored value is nonzero: bits != 0, and for float32 / float64
 * the bits without the sign (-0.0 is not selected, NaN is).  The view's C-order positions are cut into runs of run_len
 * positions (run_len divides the view's size: a rank's part of a C-order array is such a set of runs), and every run
 * into chunks of at most RB200_COMPACT_CHUNK positions; chunk c of run r is number q = c * n_runs + r, with
 * cpr = ceil(run_len / RB200_COMPACT_CHUNK) chunks per run.
 *   rb200_compact_count writes counts[q], the selected elements of chunk q (device, n_runs * cpr int64).
 *   rb200_compact writes the payload of every selected element of chunk q, in C order, from position
 *     run_base[r] + incl[q] - counts[q], where incl is the inclusive scan of counts along each run (for cpr == 1, incl
 *     may be counts itself; rb200_cumulative over [cpr][n_runs] with n_inner = n_runs gives it otherwise).
 *   Payload forms: RB200_COMPACT_VALUES: the element of `values` (same shape as cond, 1/2/4/8-byte elements) at the
 *     same position, out[0] elem_bytes per element; RB200_COMPACT_FLAT: sum((origin[d] + c_d) * gstride[d]), out[0] int64;
 *     RB200_COMPACT_COORDS: origin[d] + c_d into out[d] for every dim d of the view (int64 each).
 * cond_dtype: any storage dtype matching cond->elem_bytes.  origin / gstride: host arrays of cond->ndim entries, out: a
 * host array of device pointers; all read during the call.  Positions depend only on the data.  No scratch.  Malformed
 * arguments are rejected with a reason before any device query.                                                       */
#define RB200_COMPACT_CHUNK 4096
enum rb200_compact_form { RB200_COMPACT_VALUES = 0, RB200_COMPACT_FLAT = 1, RB200_COMPACT_COORDS = 2 };

int rb200_compact_count(const rb200_index_view* cond, int32_t cond_dtype, int64_t run_len, int64_t* counts, void* stream);
int rb200_compact(const rb200_index_view* cond, int32_t cond_dtype, int64_t run_len, const int64_t* counts, const int64_t* incl,
                  const int64_t* run_base, int32_t form, const rb200_index_view* values, const int64_t* origin, const int64_t* gstride,
                  void* const* out, void* stream);
/* One text line: runs, run length, chunks per run, runs per CTA (a CTA covers one chunk or several whole short runs),
 * CTAs, and whether the condition is read with 16-byte vector loads.  Needs no device.  NULL on a malformed argument (reason in rb200_last_error); the text stays valid until
 * the next call on this thread.                                                                                       */
const char* rb200_describe_compact_plan(const rb200_index_view* cond, int64_t run_len);

/* ---- binning (histogram, bincount, digitize, searchsorted) -----------------------------------------------------------
 * rb200_histogram bins every element of the source view into B bins described by an rb200_bin_table:
 *   RB200_BINS_UNIFORM: NumPy's equal-bins path (numpy/lib/_histograms_impl.py::histogram) on each element x: it is kept
 *     when first <= x (compared in lo_dtype) and x <= last (in hi_dtype); x is converted to edge_dtype (xe), then
 *     i = trunc(((xe - first) / denom) * B), the subtraction rounded in sub_dtype and the division and product in
 *     div_dtype, with no contraction; i == B becomes B - 1; then i -= 1 when xe < edges[i], and i += 1 when
 *     i != B - 1 and xe >= edges[i + 1].  An index that leaves [0, B) is counted in *bad.
 *   RB200_BINS_EDGES: x (converted to edge_dtype, the comparison dtype) lands in bin i when edges[i] <= x < edges[i + 1],
 *     the last bin closed, in NumPy's sort order (NaN after every number); other values are dropped.
 *   RB200_BINS_INTEGER: the bin is x itself (an integer source); an element outside [0, B) is counted in *bad.
 * Without weights, out receives B int64 counts; with weights (a view of the source's shape, F64 / F32 / I64 / I32) it
 * receives B float64 sums of the weights converted to float64.  src_dtype: F64, F32, I64 or I32 (INTEGER: I64 or I32).
 * *bad (device, may be NULL when the form cannot produce one) is added to, never reset.
 * Forms (rb200_describe_hist_plan): CTA c covers the C-order positions [c * chunk, (c + 1) * chunk), chunk a function of
 * the view's size only.  `shared`: per-CTA bins in shared memory; `global`: counts too many for shared memory, added
 * with int64 atomics; `slab`: weights too many for shared memory, one pass of the shared form per slab of bins.
 * Fold order of a weighted bin (a function of the view's shape, B, the form and the source's element size only): inside
 * a CTA each warp keeps its own row; the warp takes steps of 32 lanes * E elements (E = 16 / element bytes) in
 * position order, and for each element slot of a step the weights of the lanes in one bin are added in ascending lane
 * order and that sum is added to the row; the CTA's rows are added in warp order starting from +0.0, and the CTA sums
 * in CTA order starting from +0.0.  No float atomics.  An empty bin, or one holding only -0.0, is +0.0.
 * scratch: rb200_histogram_scratch_bytes() bytes (may be NULL when that is 0).                                        */
enum rb200_bins_form { RB200_BINS_UNIFORM = 0, RB200_BINS_EDGES = 1, RB200_BINS_INTEGER = 2 };
enum rb200_search_side { RB200_SEARCH_LEFT = 0, RB200_SEARCH_RIGHT = 1 };

typedef struct rb200_bin_table {
  int32_t form;         /* rb200_bins_form                                                                        */
  int32_t edge_dtype;   /* UNIFORM: F64 or F32; EDGES: F64, F32 or I64                                           */
  int64_t n_bins;       /* B, 1 .. 2^31 - 1                                                                       */
  const void* edges;    /* device, B + 1 entries of edge_dtype, non-decreasing (UNIFORM, EDGES)                   */
  int32_t lo_dtype;     /* UNIFORM: F64, F32 or I64                                                               */
  int32_t hi_dtype;
  int32_t sub_dtype;    /* UNIFORM: F64 or F32, not narrower than edge_dtype                                      */
  int32_t div_dtype;    /* UNIFORM: F64 or F32, not narrower than sub_dtype                                       */
  double lo, hi;        /* UNIFORM: first and last for F64 / F32 comparisons (F32: a float32 value)               */
  int64_t lo_i, hi_i;   /* UNIFORM: first and last for I64 comparisons                                            */
  double first;         /* UNIFORM: first in sub_dtype                                                            */
  double denom;         /* UNIFORM: NumPy's last - first in div_dtype                                             */
} rb200_bin_table;

int rb200_histogram(const rb200_index_view* src, int32_t src_dtype, const rb200_index_view* weights, int32_t weights_dtype,
                    const rb200_bin_table* table, void* out, uint64_t* bad, void* scratch, void* stream);
int64_t rb200_histogram_scratch_bytes(const rb200_index_view* src, int32_t weighted, const rb200_bin_table* table);
/* One text line: form, chunk, CTAs, warps, shared bytes, passes, where the edge table is read and scratch.  Needs no
 * device.  NULL on a malformed argument (reason in rb200_last_error); valid until the next call on this thread.       */
const char* rb200_describe_hist_plan(const rb200_index_view* src, int32_t weighted, const rb200_bin_table* table);

/* out[p] (device, contiguous, one int64 per element in the view's C order) = the number of entries of the sorted table
 * (device, n_sorted entries of sorted_dtype F64, F32 or I64, the comparison dtype) that are below x (side LEFT) or not
 * above x (side RIGHT), x converted to sorted_dtype, in NumPy's order (NaN after every number): NumPy's searchsorted.
 * src_dtype: F64, F32, I64 or I32.                                                                                    */
int rb200_bin_search(const rb200_index_view* src, int32_t src_dtype, const void* sorted, int64_t n_sorted, int32_t sorted_dtype, int32_t side,
                     int64_t* out, void* stream);

/* ---- order statistics (median, percentile, quantile) -------------------------------------------------------------------
 * Key map.  Every element x maps to an unsigned key of KB bits (KB = 64 for F64 and I64, 32 for F32 and I32; a 32-bit
 * key is held in the low half of a uint64) whose unsigned order is NumPy's sort order:
 *   F64 / F32: every NaN, of any sign or payload, maps to 2^KB - 1 (after +inf); otherwise, with u the bits of x, a
 *              clear sign bit is set (u | 2^(KB-1)) and a set sign bit flips every bit (~u).  -0.0 sorts before +0.0.
 *   I64 / I32: the two's-complement bits with the sign bit flipped.
 * The inverse takes a key back to the value it came from (a NaN key to the default quiet NaN).
 * Segments.  The view's C-order positions form S = n / seg_len segments of seg_len consecutive positions (the reduced
 * axis is the view's last dim; seg_len = n for one segment).  Each segment has K targets, each a rank in [0, seg_len):
 * the target's key is the rank-th smallest key of its segment, counting equal keys one by one.
 * Two forms (rb200_describe_select_plan picks one from the shapes only; RB200_NO_SELECT_ROW in the environment, read at
 * each call, takes `row` out of the selection):
 *   `row`  (seg_len keys fit in shared memory): rb200_select_rows.  One CTA loads its segment once, counts its NaN keys
 *          c, and finds each target's key by 8-bit digits in shared memory; the target's rank is
 *          rank_table[(skip_nan ? seg_len - c : 0) * K + k] (rank_table, device int64: (seg_len + 1) * K entries with
 *          skip_nan, K otherwise).
 *   `pass` (otherwise): the caller runs `passes` rounds of rb200_select_count then rb200_select_choose, for p = 0, 1, ...
 *          Pass p counts the digit of `digit` bits (fewer in the last pass) below the bits chosen so far: bits
 *          [shift_p, hi_p) with hi_p = KB - p * digit and shift_p = max(hi_p - digit, 0).  The keys of a segment that
 *          match one of its count rows' prefixes (the chosen bits; pass 0: one row, every key) are counted per row
 *          into counts[(s * K + row) * 2^digit + digit value] (int64, overwritten); pass 0 also writes nans[s], the NaN
 *          keys of segment s (float sources).  With several ranks the caller sums counts (and nans) over the ranks
 *          before the choose.  rb200_select_choose then, for each target k of each segment in order, finds the bucket
 *          holding its residual rank in its row's counts, subtracts the keys of the lower buckets from rank[s*K+k] and
 *          adds the bucket's bits to key[s*K+k] (pass 0 starts from 0); the targets whose keys are equal share one
 *          count row for the next pass (n_slots[s] rows, slot[s*K+k] the target's row, slot_key its prefix), and
 *          matched[s] is the number of keys that match a row of segment s.  After the last choose key[s*K+k] is the
 *          target's key.  Before pass 0 the caller writes the ranks into rank[].
 *          Candidate compaction (one segment only): mode APPEND reads the view as READ does and also appends every key
 *          that matches a count row to cand (in no particular order: the order of keys does not change their ranks),
 *          counting them in *cand_n (the caller zeroes it first); mode CAND reads those *cand_n keys instead of the
 *          view.  The caller may switch to APPEND once matched[0] <= cand_cap (rb200_select_scratch_bytes / 8).
 *          Worst case: every key in one bucket of every digit (e.g. all keys equal): no compaction, one full read of
 *          the view per pass.                                                                                         */
enum rb200_select_mode { RB200_SELECT_READ = 0, RB200_SELECT_APPEND = 1, RB200_SELECT_CAND = 2 };

typedef struct rb200_select_state {
  int64_t segments;      /* S                                                                                        */
  int64_t targets;       /* K (per segment)                                                                          */
  int64_t* rank;         /* device, S * K: the ranks before pass 0, the residual ranks after each choose             */
  uint64_t* key;         /* device, S * K: the chosen bits; the targets' keys after the last choose                  */
  int64_t* slot;         /* device, S * K: the target's count row                                                    */
  uint64_t* slot_key;    /* device, S * K: each count row's prefix                                                   */
  int64_t* n_slots;      /* device, S                                                                                */
  int64_t* counts;       /* device, S * K * 2^digit                                                                  */
  int64_t* nans;         /* device, S                                                                                */
  int64_t* matched;      /* device, S                                                                                */
  uint64_t* cand;        /* device, cand_cap keys (APPEND / CAND)                                                    */
  int64_t cand_cap;
  int64_t* cand_n;       /* device, 1 (APPEND / CAND)                                                                */
  int32_t seg_dims;      /* 0: segment s of the view is row s of the state; else the view's segments, in C order over  */
  int64_t seg_shape[RB200_MAX_DIMS];   /* seg_shape[0..seg_dims), are rows seg_base + sum(c_d * seg_gstride[d]) (a     */
  int64_t seg_gstride[RB200_MAX_DIMS]; /* rank's block of the segments of an array cut across ranks)                  */
  int64_t seg_base;
} rb200_select_state;

int rb200_select_count(const rb200_index_view* src, int32_t src_dtype, int64_t seg_len, const rb200_select_state* state, int32_t pass,
                       int32_t mode, void* stream);
int rb200_select_choose(const rb200_index_view* src, int32_t src_dtype, int64_t seg_len, const rb200_select_state* state, int32_t pass,
                        void* stream);
/* keys: device, S * K; nans: device, S (the NaN keys of each segment).                                                */
int rb200_select_rows(const rb200_index_view* src, int32_t src_dtype, int64_t seg_len, int64_t targets, const int64_t* rank_table,
                      int32_t skip_nan, uint64_t* keys, int64_t* nans, void* stream);
/* segments = 0: the view is every segment it holds, and the form is chosen from the shapes.  segments > 0: the view holds
 * parts of `segments` segments of an array spread over ranks; the form is `pass` and the digit width and the
 * compaction rule follow the total.  rb200_select_count and rb200_select_choose plan with segments = state->segments.
 * The compaction buffer's bytes (cand_cap keys of 8 bytes: max(n / 32, 65536) keys, at most n, for one segment; 0 for
 * `row` and for several segments); -1 on a malformed argument.                                                        */
int64_t rb200_select_scratch_bytes(const rb200_index_view* src, int32_t src_dtype, int64_t seg_len, int64_t targets, int64_t segments);
/* One text line: form, digit width, passes, CTAs, chunk, count rows per launch (groups of them), shared bytes, count
 * bytes and scratch bytes.  Needs no device.  NULL on a malformed argument (reason in rb200_last_error).             */
const char* rb200_describe_select_plan(const rb200_index_view* src, int32_t src_dtype, int64_t seg_len, int64_t targets, int64_t segments);

/* Which kernel rb200_run_deferred_ops would run `op` on and how (staged views, halos, TMA or cp.async loader, ring depth,
 * lean instructions, CTAs), as one text line in out[0..cap).  Needs no device and touches no pointer: the counterpart
 * of RAMBA_SHOW_CODE printing the generated kernel (ramba/ramba.py:8266-8284).                                       */
int rb200_describe_plan(const rb200_fused_op* op, char* out, int64_t cap);

/* Thread-local description of the last error returned on this thread.               */
const char* rb200_last_error(void);

/* RB200_ABI_VERSION the library was built with.                                     */
int rb200_abi_version(void);

/* Number of kernels this library has launched since load / last reset (bench.py's
 * gpu_launches claim).                                                              */
int64_t rb200_launch_count(void);
void rb200_reset_launch_count(void);

/* Device properties used for grid sizing: returns SM count of the current device,
 * or -1 when no CUDA device is usable.                                              */
int rb200_device_sm_count(void);

#ifdef __cplusplus
}
#endif
#endif /* RAMBA_B200_H */
