// Index logic of the wgmma linear kernel (csrc/cuda/tc_gemm.cu) as plain __host__ __device__ code: how a problem becomes
// tiles, tensor maps and kernel arguments, which TMA boxes a k-block needs, where an accumulator element goes.  The kernel
// calls these functions; csrc/tests/tc_emu_test.cc compiles the same header with g++ and runs every mode of the kernel
// (both orientations, MN-major operands, split-K, cross-rank adds, reduce-scatter, all-gather) on an emulated TMA / MMA /
// accumulator — everything except the hardware's descriptor semantics, which csrc/tests/tc_desc_test.cc pins against CuTe.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include "bnet/bnet_tc.h"

#if defined(__CUDACC__)
#define BNET_TC_HD __host__ __device__ __forceinline__
#else
#define BNET_TC_HD inline
#endif

namespace bnet {
namespace tc {

constexpr int kBM = 128;               // accumulator rows of a tile: two consumer warpgroups x wgmma M = 64
constexpr int kBK = 64;                // 64 bf16 = 128 bytes = one swizzle-128B row
constexpr int kMmaK = 16;              // wgmma K, fixed for 16-bit inputs
constexpr int kABytes = kBM * kBK * 2; // lane-operand bytes per stage
constexpr int kAtomBytes = 64 * kBK * 2; // one [64 x 64] box of an MN-major operand
constexpr int kEpiPitch = 40;          // floats per row of a warp's epilogue scratch (16 rows x 32 columns)
constexpr int kEpiScratchBytes = 8 * 16 * kEpiPitch * 4;   // the 8 consumer warps' scratch

BNET_TC_HD constexpr int stages_for(int bn) { return bn <= 64 ? 6 : (bn <= 128 ? 5 : 4); }
// dynamic shared memory of a launch: the stage ring + alignment slack + epilogue scratch + 2 mbarriers per stage + fix-up slot
BNET_TC_HD constexpr int smem_bytes_for(int stages, int bn) {
  return stages * (kABytes + bn * kBK * 2) + 1024 + kEpiScratchBytes + 2 * stages * 8 + 16;
}

// ---- bf16 without cuda_bf16.h (the header is also compiled by g++)
BNET_TC_HD float bf16_to_f32(uint16_t v) {
  uint32_t u = uint32_t(v) << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}
BNET_TC_HD uint16_t f32_to_bf16(float f) {        // round to nearest even, NaN stays NaN (== __float2bfloat16_rn)
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return uint16_t((u >> 16) | 0x40);
  u += 0x7fffu + ((u >> 16) & 1);
  return uint16_t(u >> 16);
}

// 3x3 / stride 1 / pad 1 convolution as an implicit GEMM (NHWC activations, [Cout][3][3][Cin] filters = the
// channels_last memory of a torch Conv2d weight):
//     out[pixel, co] = sum over (tap, ci) of  in[pixel shifted by tap, ci] * w[co, tap, ci]
// The lane operand's 128 rows are a PATCH of output pixels: bw x bh pixels of bn images (bw * bh * bn == 128).  For
// reduction block kb = tap * cpb + cb the patch's input values are ONE 4-D TMA box {64 channels, bw, bh, bn} at
// (cb * 64, w0 + dw[tap], h0 + dh[tap], n0): out-of-bounds coordinates (the padding, ragged patches) are zero-filled by
// the TMA unit, and the box lands in shared memory as the same [128 rows x 128 bytes] swizzled image a 2-D box would
// write, so the MMA side does not know it is a convolution.  The column operand is the filter matrix [Cout][9 * Cin]:
//   forward  K-major,  k-block kb starts at column kb * 64 (tap-major, then ci)
//   dgrad    the roles of Cin / Cout swap and the taps flip: filters are read MN-major (reduction = co, outer):
//            one [64 co x 64 ci] box per 64 output columns at (tap * Cin + ci0, cb * 64)
struct ConvGeom {
  int N, H, W;               // output (== input) image batch / height / width
  int bw, bh, bn;            // patch: bw * bh * bn == 128
  int tiles_w, tiles_h, tiles_n;
  int cpb;                   // 64-channel blocks of the reduction per tap
  int col_pitch;             // dgrad: elements between taps in a filter row (= Cin of the forward layer)
  signed char dh[9], dw[9];  // input offset of tap t relative to the output pixel
};

struct TcArgs {
  ConvGeom conv;             // (only read by the convolution instantiations)
  int rows_a, rows_b;        // valid rows of the lane / column operand
  int tiles_a, n_tiles;      // 128-row blocks of the lane operand; output tiles in total (tile t = (t % tiles_a, t / tiles_a))
  int k_blocks;              // ceil(reduction / 64)
  int k_per_split;           // K blocks handled by one grid.z slice
  int ldo;                   // elements between output rows
  int act;
  const uint16_t* bias;      // bf16, indexed by the output FEATURE (column of out), may be null
  void* outs[BNET_TC_MAX_OUTS];
  int n_outs;                // reduce mode: how many output mappings (1 when multicast)
  int multicast;
  int gather_rows;           // > 0: the batch operand is split over batch maps, gather_rows rows each (all-gather fused
                             //      into the operand loads: rank p's shard is read from its memory over NVLink by TMA)
  int scatter_rows;          // > 0 (reduce mode): batch row m belongs to rank m / scatter_rows — the tile is added into
                             //      THAT rank's output only, at local row m % scatter_rows (reduce-scatter epilogue)
  int* err;
  // split-K with the finish fused into the kernel ("fix-up"): outs[0] is an fp32 workspace that is all zero on entry; the
  // K slices add their partial tiles into it in slice order (slice z waits until fix_counters[tile] == z: the same sums on
  // every run; fix_counters[n_tiles] hands out the slices' positions), count themselves in fix_counters[tile], and the slice
  // that arrives last
  // reads the sums back (they sit in L2), applies bias / activation, writes the bf16 result and re-zeroes what it read —
  // one launch, no memset, no separate epilogue pass.  fix_out == nullptr: plain reduce mode.
  void* fix_out;
  int* fix_counters;
  int fix_ldo;
};

// One GEMM operand: `rows` entries along its MN dimension (the one that survives), the reduction along the other.
//   K-major  (mn = 0): element (i, r) at ptr[i * ld + r]
//   MN-major (mn = 1): element (i, r) at ptr[r * ld + i]
struct Operand { const void* ptr; int rows; int ld; int mn; };

// What cuTensorMapEncodeTiled is told (2-D, bf16, 128-byte swizzle, zero fill outside): dim0 is the contiguous one.
struct MapDesc { const void* ptr; long long dim0, dim1; long long pitch_elems; int box0, box1; };

// ---- tiling --------------------------------------------------------------------------------------------------------------
// D[batch, feat]: `batch_rows` decides the orientation (<= 64: features ride the 128 accumulator rows, "swap").
inline int plan_gemm(int batch_rows, int feat_rows, int red, int reduce, int splits, int sm_count, BnetTcPlan* p) {
  const int M = batch_rows, N = feat_rows;
  p->swap = M <= 64 ? 1 : 0;
  p->bn = p->swap ? (M <= 32 ? 32 : 64) : 128;
  // 128 x 256 tiles (128 accumulator registers per consumer thread) once they still fill every SM: half the MMA issues and
  // 1.5x the arithmetic intensity per shared-memory byte of a 128 x 128 tile
  if (!p->swap && (long long)((N + 255) / 256) * ((M + kBM - 1) / kBM) >= sm_count) p->bn = 256;
  p->stages = stages_for(p->bn);
  const int rows_a = p->swap ? N : M, rows_b = p->swap ? M : N;
  p->grid_x = (rows_b + p->bn - 1) / p->bn;
  p->grid_y = (rows_a + kBM - 1) / kBM;
  p->k_blocks = (red + kBK - 1) / kBK;
  int z = (reduce && splits > 1) ? splits : 1;
  if (z > p->k_blocks) z = p->k_blocks;
  p->k_per_split = (p->k_blocks + z - 1) / z;
  p->grid_z = (p->k_blocks + p->k_per_split - 1) / p->k_per_split;   // no empty slices
  p->smem_bytes = smem_bytes_for(p->stages, p->bn);
  if (p->grid_z > 65535 || (long long)p->grid_x * p->grid_y > 0x7fffffffLL) return -1;
  // persistent once there are more tiles than SMs: one CTA per SM (shared memory allows no second one anyway)
  const int n_tiles = p->grid_x * p->grid_y;
  const int per_slice = sm_count / p->grid_z > 0 ? sm_count / p->grid_z : 1;
  p->ctas = n_tiles < per_slice ? n_tiles : per_slice;
  return 0;
}

inline MapDesc map_desc(const Operand& o, int red, int box_mn) {
  MapDesc d;
  d.ptr = o.ptr;
  d.dim0 = o.mn ? o.rows : red;
  d.dim1 = o.mn ? red : o.rows;
  d.pitch_elems = o.ld;
  d.box0 = kBK;
  d.box1 = o.mn ? kBK : box_mn;
  return d;
}

// Everything a launch needs, derived from the problem alone (no CUDA calls): the host wrapper encodes the MapDescs
// into CUtensorMaps and picks the template instantiation from (plan.bn, plan.swap, reduce, a_mn, b_mn).
struct Problem {
  BnetTcPlan plan;
  TcArgs args;
  MapDesc batch_maps[BNET_TC_MAX_PEERS];
  int n_batch_maps;
  MapDesc feat_map;
  bool a_mn, b_mn;           // major of the LANE / COLUMN operand (after the orientation was chosen)
};

// `shards` (optional): the batch operand's row blocks live in n_shards separate allocations of batch.rows / n_shards rows
// each; `scatter_ranks` > 0 (reduce mode): outs[r] receives only the rows rank r owns.  Returns nullptr or an error text.
inline const char* setup_problem(const Operand& batch, const Operand& feat, int red, const void* bias, void* const* outs,
                                 int n_outs, int multicast, bool reduce, int ldo, int act, int splits, int* err_dev,
                                 const void* const* shards, int n_shards, int scatter_ranks, int sm_count, Problem* pr) {
  if (batch.rows < 1 || feat.rows < 1 || red < 1) return "bad problem size";
  if (plan_gemm(batch.rows, feat.rows, red, reduce ? 1 : 0, splits, sm_count, &pr->plan) != 0) return "problem too large for one launch";
  if (!err_dev) return "err_dev is required";
  if (n_outs < 1 || n_outs > BNET_TC_MAX_OUTS) return "n_outs out of range";
  const BnetTcPlan& p = pr->plan;
  TcArgs& a = pr->args;
  memset(&a, 0, sizeof(a));
  const Operand& oa = p.swap ? feat : batch;     // lane operand: 128-row tiles
  const Operand& ob = p.swap ? batch : feat;     // column operand: bn-row tiles
  pr->a_mn = oa.mn != 0;
  pr->b_mn = ob.mn != 0;
  if (pr->b_mn && p.bn % 64) return "an MN-major column operand needs tiles of 64 or more columns";
  const int batch_box = p.swap ? p.bn : kBM;     // rows of one box of the batch operand
  if (n_shards > 0) {
    if (n_shards > BNET_TC_MAX_PEERS || batch.rows % n_shards) return "bad shard count";
    a.gather_rows = batch.rows / n_shards;
    if (a.gather_rows % batch_box) return "rows per shard must be a multiple of the tile height (128)";
    for (int r = 0; r < n_shards; r++) {
      Operand o = batch;
      o.ptr = shards[r];
      o.rows = a.gather_rows;
      pr->batch_maps[r] = map_desc(o, red, batch_box);
    }
    pr->n_batch_maps = n_shards;
  } else {
    pr->batch_maps[0] = map_desc(batch, red, batch_box);
    pr->n_batch_maps = 1;
  }
  pr->feat_map = map_desc(feat, red, p.swap ? kBM : p.bn);
  if (scatter_ranks > 0) {
    if (!reduce || multicast || n_outs != scatter_ranks || batch.rows % scatter_ranks) return "bad reduce-scatter arguments";
    a.scatter_rows = batch.rows / scatter_ranks;
  }
  a.rows_a = oa.rows; a.rows_b = ob.rows; a.tiles_a = p.grid_y; a.n_tiles = p.grid_x * p.grid_y;
  a.k_blocks = p.k_blocks; a.k_per_split = p.k_per_split; a.ldo = ldo; a.act = act;
  a.bias = static_cast<const uint16_t*>(bias);
  for (int i = 0; i < n_outs; i++) a.outs[i] = outs[i];
  a.n_outs = n_outs; a.multicast = multicast; a.err = err_dev;
  return nullptr;
}

// ---- per tile ------------------------------------------------------------------------------------------------------------
struct TileCoord {
  int a_row0, b_row0;        // first row of the tile in the lane / column operand (global: what the epilogue needs)
  int a_map, b_map;          // which batch map serves the operand that is the batch (0 unless gathered)
  int a_ld0, b_ld0;          // first row INSIDE that map (== a_row0 / b_row0 unless gathered)
};

template <int BN, bool kSwap>
BNET_TC_HD TileCoord tile_coord(const TcArgs& args, int t) {
  TileCoord c;
  c.a_row0 = (t % args.tiles_a) * kBM;
  c.b_row0 = (t / args.tiles_a) * BN;
  c.a_map = c.b_map = 0;
  c.a_ld0 = c.a_row0;
  c.b_ld0 = c.b_row0;
  if (args.gather_rows > 0) {
    // the tile's batch rows come from ONE rank's shard (gather_rows is a multiple of the tile height)
    if (kSwap) { c.b_map = c.b_row0 / args.gather_rows; c.b_ld0 = c.b_row0 % args.gather_rows; }
    else       { c.a_map = c.a_row0 / args.gather_rows; c.a_ld0 = c.a_row0 % args.gather_rows; }
  }
  return c;
}

// The TMA boxes of one k-block.  ld(operand /*0 = lane, 1 = column*/, byte offset inside the operand's stage area, c0, c1):
// c0 is the coordinate along the map's contiguous dimension.  K-major: one [rows x 64] box; MN-major: one [64 x 64] box per
// 64 MN elements, 8 KiB apart (the layout the MN-major shared-memory descriptor describes).
template <int BN, bool kAMn, bool kBMn, class F>
BNET_TC_HD void stage_loads(const TileCoord& c, int r0, F&& ld) {
  if (!kAMn) {
    ld(0, 0, r0, c.a_ld0);
  } else {
    for (int h = 0; h < kBM / 64; h++) ld(0, h * kAtomBytes, c.a_ld0 + 64 * h, r0);
  }
  if (!kBMn) {
    ld(1, 0, r0, c.b_ld0);
  } else {
    for (int h = 0; h < BN / 64; h++) ld(1, h * kAtomBytes, c.b_ld0 + 64 * h, r0);
  }
}

// ---- convolution: tile decode, TMA boxes of a k-block, accumulator row -> output pixel ---------------------------------
struct ConvTile { int w0, h0, n0, b_row0; };

template <int BN>
BNET_TC_HD ConvTile conv_tile(const TcArgs& args, int t) {
  const ConvGeom& g = args.conv;
  int ta = t % args.tiles_a;
  ConvTile c;
  c.b_row0 = (t / args.tiles_a) * BN;
  c.w0 = (ta % g.tiles_w) * g.bw;
  ta /= g.tiles_w;
  c.h0 = (ta % g.tiles_h) * g.bh;
  c.n0 = (ta / g.tiles_h) * g.bn;
  return c;
}

// lda(byte offset, c0 = channel, c1 = w, c2 = h, c3 = n): the patch box;  ldb(byte offset, c0, c1): the filter boxes
template <int BN, bool kBMn, class FA, class FB>
BNET_TC_HD void conv_stage_loads(const TcArgs& args, const ConvTile& c, int kb, FA&& lda, FB&& ldb) {
  const ConvGeom& g = args.conv;
  const int tap = kb / g.cpb, cb = kb - tap * g.cpb;
  lda(0, cb * kBK, c.w0 + g.dw[tap], c.h0 + g.dh[tap], c.n0);
  if (!kBMn) {
    ldb(0, kb * kBK, c.b_row0);
  } else {
    for (int h = 0; h < BN / 64; h++) ldb(h * kAtomBytes, tap * g.col_pitch + c.b_row0 + 64 * h, cb * kBK);
  }
}

// accumulator row r (0..127) of a patch -> row of the [N*H*W, C] output matrix, or -1 when the pixel is outside the image
BNET_TC_HD long long conv_out_row(const TcArgs& args, const ConvTile& c, int r) {
  const ConvGeom& g = args.conv;
  const int wi = r % g.bw, hi = (r / g.bw) % g.bh, ni = r / (g.bw * g.bh);
  const int w = c.w0 + wi, h = c.h0 + hi, n = c.n0 + ni;
  if (w >= g.W || h >= g.H || n >= g.N) return -1;
  return ((long long)n * g.H + h) * g.W + w;
}

// the patch that wastes the fewest accumulator rows (ties: the widest), bw * bh * bn == 128, all powers of two
inline void conv_pick_patch(int N, int H, int W, int* bw, int* bh, int* bn) {
  long long best = -1;
  for (int w = 1; w <= 128; w *= 2)
    for (int h = 1; w * h <= 128; h *= 2) {
      const int n = 128 / (w * h);
      if (w > 256 || h > 256 || n > 256) continue;
      const long long tiles = (long long)((W + w - 1) / w) * ((H + h - 1) / h) * ((N + n - 1) / n);
      if (best < 0 || tiles < best || (tiles == best && w > *bw)) { best = tiles; *bw = w; *bh = h; *bn = n; }
    }
}

// What cuTensorMapEncodeTiled is told about an NHWC activation: dims {C, W, H, N}, boxes {64, bw, bh, bn}
struct MapDesc4 { const void* ptr; int C, W, H, N; int bw, bh, bn; };

struct ConvProblem {
  BnetTcPlan plan;
  TcArgs args;
  MapDesc4 x_map;
  MapDesc w_map;
  bool dgrad;
};

// out[N,H,W,Cn] = act(conv3x3(x[N,H,W,Cred], w) + bias), stride 1, pad 1 (pure: no CUDA calls).
//   dgrad == 0: w = [Cn][3][3][Cred]  (forward)
//   dgrad == 1: w = [Cred][3][3][Cn]  (the FORWARD layer's filter read MN-major with flipped taps: x is the output gradient,
//               out the input gradient; Cred = the forward layer's Cout, Cn its Cin)
inline const char* setup_conv(const void* x, const void* w, const void* bias, void* out, int N, int H, int W, int Cred, int Cn, int act,
                              int dgrad, int* err_dev, int sm_count, ConvProblem* cp) {
  if (N < 1 || H < 1 || W < 1 || Cred < 64 || Cred % 64 || Cn < 8 || Cn % 8)
    return "conv3x3: the reduction channels must be a multiple of 64 and the output channels a multiple of 8";
  if (dgrad && Cn % 64) return "conv3x3 dgrad: the input channels must be a multiple of 64";
  if (!err_dev) return "err_dev is required";
  if ((long long)N * H * W > 0x7fffffffLL) return "too many pixels for one launch";
  cp->dgrad = dgrad != 0;
  TcArgs& a = cp->args;
  memset(&a, 0, sizeof(a));
  ConvGeom& g = a.conv;
  g.N = N; g.H = H; g.W = W;
  conv_pick_patch(N, H, W, &g.bw, &g.bh, &g.bn);
  g.tiles_w = (W + g.bw - 1) / g.bw;
  g.tiles_h = (H + g.bh - 1) / g.bh;
  g.tiles_n = (N + g.bn - 1) / g.bn;
  g.cpb = Cred / 64;
  g.col_pitch = Cn;
  for (int t = 0; t < 9; t++) {
    const int kh = t / 3, kw = t % 3;
    g.dh[t] = (signed char)(dgrad ? 1 - kh : kh - 1);
    g.dw[t] = (signed char)(dgrad ? 1 - kw : kw - 1);
  }
  const int tiles_a = g.tiles_w * g.tiles_h * g.tiles_n;
  const int bn_cols = (Cn >= 256 && (long long)tiles_a * ((Cn + 255) / 256) >= sm_count) ? 256 : (Cn > 64 ? 128 : 64);
  BnetTcPlan& p = cp->plan;
  memset(&p, 0, sizeof(p));
  p.swap = 0;
  p.bn = bn_cols;
  p.stages = stages_for(bn_cols);
  p.grid_x = (Cn + bn_cols - 1) / bn_cols;
  p.grid_y = tiles_a;
  p.grid_z = 1;
  p.k_blocks = 9 * g.cpb;
  p.k_per_split = p.k_blocks;
  p.smem_bytes = smem_bytes_for(p.stages, bn_cols);
  const long long n_tiles = (long long)p.grid_x * p.grid_y;
  if (n_tiles > 0x7fffffffLL) return "too many tiles";
  p.ctas = n_tiles < sm_count ? (int)n_tiles : sm_count;
  a.rows_a = N * H * W;
  a.rows_b = Cn;
  a.tiles_a = tiles_a;
  a.n_tiles = (int)n_tiles;
  a.k_blocks = p.k_blocks;
  a.k_per_split = p.k_per_split;
  a.ldo = Cn;
  a.act = act;
  a.bias = static_cast<const uint16_t*>(bias);
  a.outs[0] = out;
  a.n_outs = 1;
  a.err = err_dev;
  cp->x_map = MapDesc4{x, Cred, W, H, N, g.bw, g.bh, g.bn};
  MapDesc& wd = cp->w_map;
  wd.ptr = w;
  wd.pitch_elems = 9LL * (dgrad ? Cn : Cred);
  wd.dim0 = wd.pitch_elems;
  wd.dim1 = dgrad ? Cred : Cn;
  wd.box0 = kBK;
  wd.box1 = dgrad ? kBK : bn_cols;
  return nullptr;
}

// ---- convolution weight gradient ---------------------------------------------------------------------------------------
//     dw[co, tap, ci] = sum over pixels p of  gy[p, co] * x[p shifted by tap, ci]
// A GEMM whose REDUCTION runs over the pixels: D[i = co, j = tap * Cin + ci], both operands MN-major (reduction outer), the
// output matrix [Cout][9 * Cin] IS the filter gradient in torch's channels_last layout.  One k-block = a patch of 64 pixels
// (bw x bh pixels of bn images, bw * bh * bn == 64):
//   lane operand   gy: one 4-D box {64 co, bw, bh, bn} per 64 output channels of the tile at (co0 + 64 h, w0, h0, n0)
//   column operand x : one 4-D box {64 ci, bw, bh, bn} per 64 columns; every 64-column atom decodes its OWN (tap, ci0) —
//                      Cin is a multiple of 64, so an atom never straddles two taps, and a tile may (9 * Cin need not be
//                      a multiple of the tile width) — at (ci0, w0 + dw[tap], h0 + dh[tap], n0)
// A box lands in shared memory as [64 pixel rows x 128 bytes], exactly the [64 reduction rows x 64 MN elements] atom the
// MN-major shared-memory descriptor describes (the layout the linear layer's dW = gY^T . X already uses).  Padding, ragged
// patches, channels past Cout and columns past 9 * Cin are all the TMA unit's zero fill.  The pixel blocks are split over
// grid.z (split-K with the fix-up: TcArgs::fix_out), because Cout x 9 Cin alone rarely fills 132 SMs.
template <int BN, class FA, class FB>
BNET_TC_HD void wgrad_stage_loads(const TcArgs& args, const TileCoord& c, int kb, FA&& lda, FB&& ldb) {
  const ConvGeom& g = args.conv;
  int t = kb;
  const int w0 = (t % g.tiles_w) * g.bw;
  t /= g.tiles_w;
  const int h0 = (t % g.tiles_h) * g.bh;
  const int n0 = (t / g.tiles_h) * g.bn;
  for (int h = 0; h < kBM / 64; h++) lda(h * kAtomBytes, c.a_row0 + 64 * h, w0, h0, n0);
  for (int h = 0; h < BN / 64; h++) {
    const int col = c.b_row0 + 64 * h;
    int tap = col / g.col_pitch, ci0 = col - tap * g.col_pitch;
    if (tap >= 9) { tap = 0; ci0 = g.col_pitch; }          // past the last filter column: a box outside the tensor (zeros)
    ldb(h * kAtomBytes, ci0, w0 + g.dw[tap], h0 + g.dh[tap], n0);
  }
}

// the 64-pixel patch that needs the fewest k-blocks (ties: the widest), all powers of two
inline void conv_pick_patch64(int N, int H, int W, int* bw, int* bh, int* bn) {
  long long best = -1;
  for (int w = 1; w <= 64; w *= 2)
    for (int h = 1; w * h <= 64; h *= 2) {
      const int n = 64 / (w * h);
      const long long tiles = (long long)((W + w - 1) / w) * ((H + h - 1) / h) * ((N + n - 1) / n);
      if (best < 0 || tiles < best || (tiles == best && w > *bw)) { best = tiles; *bw = w; *bh = h; *bn = n; }
    }
}

struct WgradProblem {
  BnetTcPlan plan;
  TcArgs args;
  MapDesc4 gy_map, x_map;      // boxes of {64 channels, bw, bh, bn} with bw * bh * bn == 64
};

// dw[Cout][3][3][Cin] (bf16) = filter gradient of y = conv3x3(x, w), stride 1, pad 1; gy [N,H,W,Cout], x [N,H,W,Cin] NHWC bf16.
// `ws`: fp32 [Cout][9 * Cin] workspace, `counters`: one int per output tile (>= wgrad_max_tiles), both all zero on entry and
// left all zero.  splits <= 0: as many K slices as keep the SMs busy.  Pure: no CUDA calls.
// (+ 1: the int after the tile counters is the fix-up's ticket, see tc_gemm.cu)
inline int wgrad_max_tiles(int Cin, int Cout) { return ((Cout + kBM - 1) / kBM) * ((9 * Cin + 127) / 128) + 1; }

// fixup == 0: plain reduce mode — the slices only ADD into `ws` (fp32 [Cout][9 Cin], zero on entry) and the caller converts
// it to bf16 and clears it afterwards (two small passes); the fall-back when the in-kernel finish cannot be trusted.
inline const char* setup_conv_wgrad(const void* gy, const void* x, float* ws, void* dw, int* counters, int N, int H, int W, int Cin,
                                    int Cout, int splits, int* err_dev, int sm_count, WgradProblem* wp, int force_bn = 0,
                                    int fixup = 1) {
  if (N < 1 || H < 1 || W < 1 || Cin < 64 || Cin % 64 || Cout < 64 || Cout % 64)
    return "conv3x3 wgrad: input and output channels must be multiples of 64";
  if (!err_dev || !ws || !counters) return "conv3x3 wgrad needs err_dev, a workspace and tile counters";
  if ((long long)N * H * W > 0x7fffffffLL) return "too many pixels for one launch";
  TcArgs& a = wp->args;
  memset(&a, 0, sizeof(a));
  ConvGeom& g = a.conv;
  g.N = N; g.H = H; g.W = W;
  conv_pick_patch64(N, H, W, &g.bw, &g.bh, &g.bn);
  g.tiles_w = (W + g.bw - 1) / g.bw;
  g.tiles_h = (H + g.bh - 1) / g.bh;
  g.tiles_n = (N + g.bn - 1) / g.bn;
  g.cpb = Cin / 64;
  g.col_pitch = Cin;
  for (int t = 0; t < 9; t++) {
    g.dh[t] = (signed char)(t / 3 - 1);
    g.dw[t] = (signed char)(t % 3 - 1);
  }
  const long long kblocks = (long long)g.tiles_w * g.tiles_h * g.tiles_n;
  if (kblocks > 0x3fffffffLL) return "too many pixel blocks";
  const int cols = 9 * Cin;
  // 256-column tiles (half the MMA issues per byte of gy) unless they waste more than ~1/7 of the columns (Cin = 64: 576 columns)
  const int t256 = (cols + 255) / 256, t128 = (cols + 127) / 128;
  int bn_cols = (long long)t256 * 256 * 7 <= (long long)cols * 8 ? 256 : 128;
  if (force_bn == 128 || force_bn == 256) bn_cols = force_bn;       // (BNET_TC_WGRAD_BN: the self-check's fallback ladder)
  const int tiles_b = bn_cols == 256 ? t256 : t128;
  const int tiles_a = (Cout + kBM - 1) / kBM;
  BnetTcPlan& p = wp->plan;
  memset(&p, 0, sizeof(p));
  p.swap = 0;
  p.bn = bn_cols;
  p.stages = stages_for(bn_cols);
  p.grid_x = tiles_b;
  p.grid_y = tiles_a;
  p.k_blocks = (int)kblocks;
  const int n_tiles = tiles_a * tiles_b;
  int z = splits;
  if (z <= 0) {
    // automatic: a slice runs sm_count / z persistent CTAs, so z slices finish after ceil(n_tiles / (sm_count / z)) tile
    // passes of 1 / z of the pixels each.  Take the smallest z within 5 % of the best such time — every further slice
    // adds its partial tiles into the workspace once more.
    const long long zmax = kblocks < sm_count ? kblocks : sm_count;
    auto cost = [&](long long zz) {
      const long long per = sm_count / zz > 0 ? sm_count / zz : 1;
      return double((n_tiles + per - 1) / per) / double(zz);
    };
    double best = cost(1);
    for (long long zz = 2; zz <= zmax; zz++) best = cost(zz) < best ? cost(zz) : best;
    z = 1;
    while (z < zmax && cost(z) > best * 1.05) z++;
  }
  if (z > p.k_blocks) z = p.k_blocks;
  if (z > 65535) z = 65535;
  p.k_per_split = (p.k_blocks + z - 1) / z;
  p.grid_z = (p.k_blocks + p.k_per_split - 1) / p.k_per_split;      // no empty slices
  p.smem_bytes = smem_bytes_for(p.stages, bn_cols);
  const int per_slice = sm_count / p.grid_z > 0 ? sm_count / p.grid_z : 1;
  p.ctas = n_tiles < per_slice ? n_tiles : per_slice;
  a.rows_a = Cout;
  a.rows_b = cols;
  a.tiles_a = tiles_a;
  a.n_tiles = n_tiles;
  a.k_blocks = p.k_blocks;
  a.k_per_split = p.k_per_split;
  a.ldo = cols;
  a.act = BNET_TC_ACT_NONE;
  a.bias = nullptr;
  a.outs[0] = ws;
  a.n_outs = 1;
  a.err = err_dev;
  a.fix_out = fixup ? dw : nullptr;
  a.fix_counters = fixup ? counters : nullptr;
  a.fix_ldo = cols;
  wp->gy_map = MapDesc4{gy, Cout, W, H, N, g.bw, g.bh, g.bn};
  wp->x_map = MapDesc4{x, Cin, W, H, N, g.bw, g.bh, g.bn};
  return nullptr;
}

// One epilogue step of one thread: 16 consecutive accumulator columns (j0 .. j0+15) of accumulator row i_glob.
//   kSwap:   false -> lane i = batch row m, column j = feature n; out[m, n] = out[i * ldo + j]
//            true  -> lane i = feature n,   column j = batch row m; out[m, n] = out[j * ldo + i]
//   kReduce: fp32 adds into args.outs[] (all ranks, or with scatter_rows the owner of the batch row) instead of a bf16 store
// `Out` supplies the memory operations: st16(uint16_t*, bf16 bits), st16x16(uint16_t* 16-byte aligned, const float[16]),
// add1(float*, v, multicast), add4(float* 16-byte aligned, const float[4], multicast).
template <bool kSwap, bool kReduce, class Out>
BNET_TC_HD void epilogue_chunk(const TcArgs& args, int i_glob, int j0, const float (&acc)[16], bool add_bias, Out&& out) {
  if (i_glob >= args.rows_a || j0 >= args.rows_b) return;
  float f[16];
  const float bias_i = (kSwap && add_bias) ? bf16_to_f32(args.bias[i_glob]) : 0.f;
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
  for (int u = 0; u < 16; u++) {
    const float b = kSwap ? bias_i : ((add_bias && j0 + u < args.rows_b) ? bf16_to_f32(args.bias[j0 + u]) : 0.f);
    f[u] = acc[u] + b;
    if (!kReduce && args.act == BNET_TC_ACT_RELU) f[u] = f[u] <= 0.f ? 0.f : f[u];     // (eager torch: relu(NaN) = NaN)
  }
  if (!kReduce) {
    uint16_t* o = static_cast<uint16_t*>(args.outs[0]);
    if (kSwap) {
      // out[(j0 + u) * ldo + i]: for every u the warp writes 32 consecutive features
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
      for (int u = 0; u < 16; u++)
        if (j0 + u < args.rows_b) out.st16(o + size_t(j0 + u) * args.ldo + i_glob, f32_to_bf16(f[u]));
    } else {
      uint16_t* row = o + size_t(i_glob) * args.ldo + j0;
      if (j0 + 16 <= args.rows_b && (reinterpret_cast<uintptr_t>(row) & 15) == 0) {
        out.st16x16(row, f);
      } else {
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
        for (int u = 0; u < 16; u++)
          if (j0 + u < args.rows_b) out.st16(row + u, f32_to_bf16(f[u]));
      }
    }
  } else {
    const int o_end = args.scatter_rows > 0 ? 1 : args.n_outs;
    for (int oi = 0; oi < o_end; oi++) {
      if (kSwap) {
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
        for (int u = 0; u < 16; u++) {
          int m = j0 + u;                      // batch row
          if (m >= args.rows_b) continue;
          int o = oi;
          if (args.scatter_rows > 0) { o = m / args.scatter_rows; m -= o * args.scatter_rows; }
          out.add1(static_cast<float*>(args.outs[o]) + size_t(m) * args.ldo + i_glob, f[u], args.multicast != 0);
        }
      } else {
        int m = i_glob, o = oi;
        if (args.scatter_rows > 0) { o = m / args.scatter_rows; m -= o * args.scatter_rows; }
        float* row = static_cast<float*>(args.outs[o]) + size_t(m) * args.ldo + j0;
        const bool vec = j0 + 16 <= args.rows_b && (reinterpret_cast<uintptr_t>(row) & 15) == 0;
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
        for (int u = 0; u < 16; u += 4) {
          if (vec) {
            out.add4(row + u, f + u, args.multicast != 0);
          } else {
            for (int e = u; e < u + 4; e++)
              if (j0 + e < args.rows_b) out.add1(row + e, f[e], args.multicast != 0);
          }
        }
      }
    }
  }
}

}  // namespace tc
}  // namespace bnet
