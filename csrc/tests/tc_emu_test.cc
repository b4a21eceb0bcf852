// The wgmma linear kernel's index logic (csrc/cuda/tc_body.cuh) on an emulated TMA / MMA / accumulator, no GPU needed.
//
// What runs here is the code the kernel runs: setup_problem (orientation, tensor-map descriptions, kernel arguments),
// tile_coord (tile -> rows, gathered shard), stage_loads (which TMA boxes, at which coordinates, where in the stage) and
// epilogue_chunk (bias / ReLU / bf16 store, cross-rank adds, reduce-scatter).  What is emulated: the TMA engine (a box
// copy with zero fill), the MMA (a dot product over the stage as the shared-memory descriptors describe it: K-major
// rows, or MN-major 64 x 64 atoms 8 KiB apart) and the register accumulator (a float array).  Every mode is compared with a
// plain GEMM.
//
//   make build/tests/tc_emu_test && build/tests/tc_emu_test
#include <math.h>
#include <stdio.h>
#include <stdlib.h>

#include <vector>

#include "cuda/tc_body.cuh"

using namespace bnet::tc;

static int g_failures = 0;
#define CHECK(cond, ...) do { if (!(cond)) { printf("FAIL %s:%d: ", __FILE__, __LINE__); printf(__VA_ARGS__); printf("\n"); g_failures++; } } while (0)

static uint32_t g_rng = 12345;
static float rnd() { g_rng = g_rng * 1664525u + 1013904223u; return float(int((g_rng >> 9) % 9) - 4) * 0.25f; }   // exact in bf16

struct Mat {   // bf16 matrix with a row pitch
  int rows, cols, ld;
  std::vector<uint16_t> v;
  Mat(int r, int c, int pad = 0) : rows(r), cols(c), ld(c + pad), v(size_t(r) * (c + pad) + 8, 0x7fc0 /* NaN in the padding */) {
    for (int i = 0; i < r; i++) for (int j = 0; j < c; j++) v[size_t(i) * ld + j] = f32_to_bf16(rnd());
  }
  float at(int i, int j) const { return bf16_to_f32(v[size_t(i) * ld + j]); }
  const void* ptr() const { return v.data(); }
};

// ---- emulated hardware ---------------------------------------------------------------------------------------------------
static void tma_box(const MapDesc& d, int c0, int c1, uint16_t* dst) {
  const uint16_t* src = static_cast<const uint16_t*>(d.ptr);
  for (int r = 0; r < d.box1; r++)
    for (int c = 0; c < d.box0; c++) {
      const long long x = c0 + c, y = c1 + r;
      dst[r * d.box0 + c] = (x >= 0 && x < d.dim0 && y >= 0 && y < d.dim1) ? src[y * d.pitch_elems + x] : 0;
    }
}

// element (i, k) of an operand's stage area, as the shared-memory descriptor of its major describes it
static float stage_at(const uint16_t* area, bool mn, int i, int k) {
  return bf16_to_f32(mn ? area[(i / 64) * (kAtomBytes / 2) + k * 64 + i % 64] : area[i * kBK + k]);
}

struct HostOut {
  float* mc_base = nullptr;                 // multicast: the pointer the kernel was given ...
  std::vector<float*> replicas;             // ... stands for these buffers (the switch replicates the add)
  void st16(uint16_t* p, uint16_t v) const { *p = v; }
  void st16x16(uint16_t* row, const float (&f)[16]) const { for (int u = 0; u < 16; u++) row[u] = f32_to_bf16(f[u]); }
  void add1(float* p, float v, bool multicast) const {
    if (!multicast) { *p += v; return; }
    for (float* r : replicas) r[p - mc_base] += v;
  }
  void add4(float* p, const float* f, bool multicast) const { for (int u = 0; u < 4; u++) add1(p + u, f[u], multicast); }
};

template <int BN, bool kSwap, bool kReduce, bool kAMn, bool kBMn>
static void run_kernel(const Problem& pr, const HostOut& out) {
  const TcArgs& args = pr.args;
  const BnetTcPlan& p = pr.plan;
  std::vector<uint16_t> stage_a(kABytes / 2), stage_b(BN * kBK);
  std::vector<float> accum(size_t(kBM) * BN);
  for (int z = 0; z < p.grid_z; z++) {
    const int kb_begin = z * args.k_per_split;
    const int kb_end = kb_begin + args.k_per_split < args.k_blocks ? kb_begin + args.k_per_split : args.k_blocks;
    CHECK(kb_end > kb_begin, "empty K slice %d", z);
    for (int cta = 0; cta < p.ctas; cta++) {
      for (int t = cta; t < args.n_tiles; t += p.ctas) {
        const TileCoord tc = tile_coord<BN, kSwap>(args, t);
        std::fill(accum.begin(), accum.end(), 0.f);
        for (int kb = kb_begin; kb < kb_end; kb++) {
          std::fill(stage_a.begin(), stage_a.end(), uint16_t(0x7fc0));     // stale data must never be read
          std::fill(stage_b.begin(), stage_b.end(), uint16_t(0x7fc0));
          int bytes = 0;
          stage_loads<BN, kAMn, kBMn>(tc, kb * kBK, [&](int operand, int offset, int c0, int c1) {
            const MapDesc& d = operand == 0 ? (kSwap ? pr.feat_map : pr.batch_maps[tc.a_map])
                                            : (kSwap ? pr.batch_maps[tc.b_map] : pr.feat_map);
            tma_box(d, c0, c1, (operand ? stage_b.data() : stage_a.data()) + offset / 2);
            bytes += d.box0 * d.box1 * 2;
          });
          CHECK(bytes == kABytes + BN * kBK * 2, "expect_tx bytes %d", bytes);
          for (int i = 0; i < kBM; i++)
            for (int j = 0; j < BN; j++) {
              float s = 0.f;
              for (int k = 0; k < kBK; k++) s += stage_at(stage_a.data(), kAMn, i, k) * stage_at(stage_b.data(), kBMn, j, k);
              accum[size_t(i) * BN + j] += s;
            }
        }
        const bool add_bias = args.bias != nullptr && (!kReduce || z == 0);
        // the kernel's consumer warps 4 .. 11: warp w takes rows 64 (w / 4 - 1) + 16 (w % 4) .. +15, and per 32-column chunk
        // lane l finishes row l % 16, columns 16 (l / 16) .. +15
        for (int warp = 4; warp < 12; warp++)
          for (int lane = 0; lane < 32; lane++) {
            const int i_local = 64 * (warp / 4 - 1) + 16 * (warp % 4) + (lane & 15);
            for (int cc = 0; cc < BN / 32; cc++) {
              const int col = 32 * cc + 16 * (lane >> 4);
              float acc[16];
              for (int u = 0; u < 16; u++) acc[u] = accum[size_t(i_local) * BN + col + u];
              epilogue_chunk<kSwap, kReduce>(args, tc.a_row0 + i_local, tc.b_row0 + col, acc, add_bias, out);
            }
          }
      }
    }
  }
}

static bool dispatch(const Problem& pr, bool reduce, const HostOut& out) {
  const BnetTcPlan& p = pr.plan;
  const bool swap = p.swap != 0, amn = pr.a_mn, bmn = pr.b_mn;
#define CASE(BN, SWAP, RED, AMN, BMN) \
  if (p.bn == BN && swap == SWAP && reduce == RED && amn == AMN && bmn == BMN) { run_kernel<BN, SWAP, RED, AMN, BMN>(pr, out); return true; }
  CASE(32, true, false, false, false)   CASE(32, true, true, false, false)
  CASE(64, true, false, false, false)   CASE(64, true, true, false, false)
  CASE(128, false, false, false, false) CASE(128, false, true, false, false)
  CASE(256, false, false, false, false) CASE(256, false, true, false, false)
  CASE(128, false, false, false, true)  CASE(256, false, false, false, true)
  CASE(32, true, false, true, false)    CASE(64, true, false, true, false)
  CASE(128, false, false, true, true)   CASE(256, false, false, true, true)
#undef CASE
  return false;
}

static bool close(float got, double want) { return fabs(got - want) <= 0.02 + 0.01 * fabs(want); }

// ---- scenarios -----------------------------------------------------------------------------------------------------------
static void forward(int M, int N, int K, bool bias, bool relu, int sms, int pad) {
  Mat x(M, K, pad), w(N, K, pad ? 8 : 0), b(1, N);
  std::vector<uint16_t> out(size_t(M) * (N + 8) + 16, 0xdead);
  uint16_t* o = out.data();
  while (reinterpret_cast<uintptr_t>(o) & 15) o++;
  void* outs[1] = {o};
  int err = 0;
  Problem pr;
  const char* e = setup_problem(Operand{x.ptr(), M, x.ld, 0}, Operand{w.ptr(), N, w.ld, 0}, K, bias ? b.ptr() : nullptr, outs, 1, 0,
                                false, N + 8, relu ? BNET_TC_ACT_RELU : 0, 1, &err, nullptr, 0, 0, sms, &pr);
  CHECK(e == nullptr, "setup: %s", e ? e : "");
  if (e) return;
  CHECK(dispatch(pr, false, HostOut{}), "no kernel for forward %dx%dx%d", M, N, K);
  int bad = 0;
  for (int m = 0; m < M; m++)
    for (int n = 0; n < N; n++) {
      double r = bias ? b.at(0, n) : 0.0;
      for (int k = 0; k < K; k++) r += double(x.at(m, k)) * w.at(n, k);
      if (relu && r < 0) r = 0;
      if (!close(bf16_to_f32(o[size_t(m) * (N + 8) + n]), r)) bad++;
    }
  for (int m = 0; m < M; m++)
    for (int n = N; n < N + 8; n++)
      if (o[size_t(m) * (N + 8) + n] != 0xdead) bad++;       // nothing written past the row
  CHECK(bad == 0, "forward M=%d N=%d K=%d bias=%d relu=%d sms=%d (swap %d bn %d ctas %d): %d wrong", M, N, K, bias, relu, sms,
        pr.plan.swap, pr.plan.bn, pr.plan.ctas, bad);
}

static void reduce(int M, int N, int K, int n_outs, bool multicast, int splits, int scatter, bool bias) {
  Mat x(M, K), w(N, K), b(1, N);
  const int rows_out = scatter ? M / scatter : M;
  const int n_bufs = scatter ? scatter : n_outs;
  std::vector<std::vector<float>> bufs(n_bufs, std::vector<float>(size_t(rows_out) * N + 4, 0.f));
  std::vector<float*> ptrs;
  for (auto& v : bufs) { float* p = v.data(); while (reinterpret_cast<uintptr_t>(p) & 15) p++; ptrs.push_back(p); }
  HostOut ho;
  void* outs[BNET_TC_MAX_OUTS];
  int n = 0;
  if (multicast) { ho.mc_base = ptrs[0]; ho.replicas = ptrs; outs[0] = ptrs[0]; n = 1; }
  else { for (float* p : ptrs) outs[n++] = p; }
  int err = 0;
  Problem pr;
  const char* e = setup_problem(Operand{x.ptr(), M, x.ld, 0}, Operand{w.ptr(), N, w.ld, 0}, K, bias ? b.ptr() : nullptr, outs, n,
                                multicast ? 1 : 0, true, N, 0, splits, &err, nullptr, 0, scatter, 132, &pr);
  CHECK(e == nullptr, "setup: %s", e ? e : "");
  if (e) return;
  CHECK(dispatch(pr, true, ho), "no kernel for reduce %dx%dx%d", M, N, K);
  int bad = 0;
  for (int m = 0; m < M; m++)
    for (int nn = 0; nn < N; nn++) {
      double r = bias ? b.at(0, nn) : 0.0;
      for (int k = 0; k < K; k++) r += double(x.at(m, k)) * w.at(nn, k);
      for (int o = 0; o < n_bufs; o++) {
        double want = r;
        int row = m;
        if (scatter) { want = (m / rows_out == o) ? r : 0.0; row = m % rows_out; if (m / rows_out != o) continue; }
        if (!close(ptrs[o][size_t(row) * N + nn], want)) bad++;
      }
    }
  CHECK(bad == 0, "reduce M=%d N=%d K=%d outs=%d mc=%d splits=%d scatter=%d (swap %d bn %d z %d): %d wrong", M, N, K, n_outs,
        multicast, splits, scatter, pr.plan.swap, pr.plan.bn, pr.plan.grid_z, bad);
}

static void gather(int shards, int rows, int N, int K) {
  std::vector<Mat> xs;
  for (int r = 0; r < shards; r++) xs.emplace_back(rows, K);
  Mat w(N, K), b(1, N);
  const int M = shards * rows;
  std::vector<uint16_t> out(size_t(M) * N + 16, 0);
  uint16_t* o = out.data();
  while (reinterpret_cast<uintptr_t>(o) & 15) o++;
  void* outs[1] = {o};
  const void* sp[BNET_TC_MAX_PEERS];
  for (int r = 0; r < shards; r++) sp[r] = xs[r].ptr();
  int err = 0;
  Problem pr;
  const char* e = setup_problem(Operand{sp[0], M, K, 0}, Operand{w.ptr(), N, w.ld, 0}, K, b.ptr(), outs, 1, 0, false, N, 0, 1, &err, sp,
                                shards, 0, 5, &pr);
  CHECK(e == nullptr, "setup: %s", e ? e : "");
  if (e) return;
  CHECK(dispatch(pr, false, HostOut{}), "no kernel for gather");
  int bad = 0;
  for (int m = 0; m < M; m++)
    for (int n = 0; n < N; n++) {
      double r = b.at(0, n);
      for (int k = 0; k < K; k++) r += double(xs[m / rows].at(m % rows, k)) * w.at(n, k);
      if (!close(bf16_to_f32(o[size_t(m) * N + n]), r)) bad++;
    }
  CHECK(bad == 0, "all-gather linear %d x %d rows, N=%d K=%d: %d wrong", shards, rows, N, K, bad);
}

static void backward(int M, int N, int K) {
  Mat gy(M, N), w(N, K), x(M, K);
  std::vector<uint16_t> dxv(size_t(M) * K + 16, 0), dwv(size_t(N) * K + 16, 0);
  uint16_t *dx = dxv.data(), *dw = dwv.data();
  while (reinterpret_cast<uintptr_t>(dx) & 15) dx++;
  while (reinterpret_cast<uintptr_t>(dw) & 15) dw++;
  int err = 0;
  Problem pr;
  void* o1[1] = {dx};
  const char* e = setup_problem(Operand{gy.ptr(), M, gy.ld, 0}, Operand{w.ptr(), K, w.ld, 1}, N, nullptr, o1, 1, 0, false, K, 0, 1, &err,
                                nullptr, 0, 0, 132, &pr);
  CHECK(e == nullptr, "dgrad setup: %s", e ? e : "");
  if (!e) {
    CHECK(dispatch(pr, false, HostOut{}), "no kernel for dgrad %dx%dx%d (swap %d bn %d)", M, N, K, pr.plan.swap, pr.plan.bn);
    int bad = 0;
    for (int m = 0; m < M; m++)
      for (int k = 0; k < K; k++) {
        double r = 0;
        for (int n = 0; n < N; n++) r += double(gy.at(m, n)) * w.at(n, k);
        if (!close(bf16_to_f32(dx[size_t(m) * K + k]), r)) bad++;
      }
    CHECK(bad == 0, "dgrad M=%d N=%d K=%d (swap %d): %d wrong", M, N, K, pr.plan.swap, bad);
  }
  if (N <= 64) return;
  void* o2[1] = {dw};
  e = setup_problem(Operand{gy.ptr(), N, gy.ld, 1}, Operand{x.ptr(), K, x.ld, 1}, M, nullptr, o2, 1, 0, false, K, 0, 1, &err, nullptr, 0, 0,
                    132, &pr);
  CHECK(e == nullptr, "wgrad setup: %s", e ? e : "");
  if (e) return;
  CHECK(dispatch(pr, false, HostOut{}), "no kernel for wgrad %dx%dx%d", M, N, K);
  int bad = 0;
  for (int n = 0; n < N; n++)
    for (int k = 0; k < K; k++) {
      double r = 0;
      for (int m = 0; m < M; m++) r += double(gy.at(m, n)) * x.at(m, k);
      if (!close(bf16_to_f32(dw[size_t(n) * K + k]), r)) bad++;
    }
  CHECK(bad == 0, "wgrad M=%d N=%d K=%d: %d wrong", M, N, K, bad);
}

// ---- convolution (implicit GEMM): 4-D boxes with zero fill, the same MMA / accumulator emulation ------------------------
static void tma_box4(const MapDesc4& d, int c0, int c1, int c2, int c3, uint16_t* dst) {
  const uint16_t* src = static_cast<const uint16_t*>(d.ptr);
  size_t o = 0;
  for (int n = 0; n < d.bn; n++)
    for (int h = 0; h < d.bh; h++)
      for (int w = 0; w < d.bw; w++)
        for (int c = 0; c < kBK; c++) {
          const long long cc = c0 + c, ww = c1 + w, hh = c2 + h, nn = c3 + n;
          const bool in = cc >= 0 && cc < d.C && ww >= 0 && ww < d.W && hh >= 0 && hh < d.H && nn >= 0 && nn < d.N;
          dst[o++] = in ? src[((nn * d.H + hh) * d.W + ww) * d.C + cc] : 0;
        }
}

template <int BN, bool kBMn>
static void run_conv_kernel(const ConvProblem& cp, const HostOut& out) {
  const TcArgs& args = cp.args;
  const BnetTcPlan& p = cp.plan;
  std::vector<uint16_t> stage_a(kABytes / 2), stage_b(BN * kBK);
  std::vector<float> accum(size_t(kBM) * BN);
  CHECK(args.conv.bw * args.conv.bh * args.conv.bn == kBM, "patch %d x %d x %d", args.conv.bw, args.conv.bh, args.conv.bn);
  for (int cta = 0; cta < p.ctas; cta++)
    for (int t = cta; t < args.n_tiles; t += p.ctas) {
      const ConvTile ct = conv_tile<BN>(args, t);
      std::fill(accum.begin(), accum.end(), 0.f);
      for (int kb = 0; kb < args.k_blocks; kb++) {
        std::fill(stage_a.begin(), stage_a.end(), uint16_t(0x7fc0));
        std::fill(stage_b.begin(), stage_b.end(), uint16_t(0x7fc0));
        int bytes = 0;
        conv_stage_loads<BN, kBMn>(args, ct, kb,
            [&](int offset, int c0, int c1, int c2, int c3) { tma_box4(cp.x_map, c0, c1, c2, c3, stage_a.data() + offset / 2); bytes += kABytes; },
            [&](int offset, int c0, int c1) { tma_box(cp.w_map, c0, c1, stage_b.data() + offset / 2); bytes += cp.w_map.box0 * cp.w_map.box1 * 2; });
        CHECK(bytes == kABytes + BN * kBK * 2, "conv expect_tx bytes %d", bytes);
        for (int i = 0; i < kBM; i++)
          for (int j = 0; j < BN; j++) {
            float s = 0.f;
            for (int k = 0; k < kBK; k++) s += stage_at(stage_a.data(), false, i, k) * stage_at(stage_b.data(), kBMn, j, k);
            accum[size_t(i) * BN + j] += s;
          }
      }
      for (int r = 0; r < kBM; r++) {
        const long long row = conv_out_row(args, ct, r);
        const int i_glob = row < 0 ? args.rows_a : (int)row;
        for (int c = 0; c < BN / 16; c++) {
          float acc[16];
          for (int u = 0; u < 16; u++) acc[u] = accum[size_t(r) * BN + c * 16 + u];
          epilogue_chunk<false, false>(args, i_glob, ct.b_row0 + c * 16, acc, args.bias != nullptr, out);
        }
      }
    }
}

static void conv(int N, int H, int W, int Cin, int Cout, bool relu, int sms) {
  // x [N,H,W,Cin], w [Cout][3][3][Cin], y [N,H,W,Cout]
  Mat x(N * H * W, Cin), w(Cout, 9 * Cin), b(1, Cout);
  std::vector<uint16_t> yv(size_t(N) * H * W * Cout + 16, 0xdead);
  uint16_t* y = yv.data();
  while (reinterpret_cast<uintptr_t>(y) & 15) y++;
  int err = 0;
  ConvProblem cp;
  const char* e = setup_conv(x.ptr(), w.ptr(), b.ptr(), y, N, H, W, Cin, Cout, relu ? BNET_TC_ACT_RELU : 0, 0, &err, sms, &cp);
  CHECK(e == nullptr, "conv setup: %s", e ? e : "");
  if (e) return;
  if (cp.plan.bn == 64) run_conv_kernel<64, false>(cp, HostOut{});
  else if (cp.plan.bn == 128) run_conv_kernel<128, false>(cp, HostOut{});
  else run_conv_kernel<256, false>(cp, HostOut{});
  int bad = 0;
  for (int n = 0; n < N; n++)
    for (int h = 0; h < H; h++)
      for (int ww = 0; ww < W; ww++)
        for (int co = 0; co < Cout; co++) {
          double r = b.at(0, co);
          for (int kh = 0; kh < 3; kh++)
            for (int kw = 0; kw < 3; kw++) {
              const int hh = h + kh - 1, w2 = ww + kw - 1;
              if (hh < 0 || hh >= H || w2 < 0 || w2 >= W) continue;
              for (int ci = 0; ci < Cin; ci++) r += double(x.at((n * H + hh) * W + w2, ci)) * w.at(co, (kh * 3 + kw) * Cin + ci);
            }
          if (relu && r < 0) r = 0;
          if (!close(bf16_to_f32(y[(size_t(n * H + h) * W + ww) * Cout + co]), r)) bad++;
        }
  CHECK(bad == 0, "conv fwd N=%d %dx%d %d->%d (patch %dx%dx%d bn %d ctas %d): %d wrong", N, H, W, Cin, Cout, cp.args.conv.bw,
        cp.args.conv.bh, cp.args.conv.bn, cp.plan.bn, cp.plan.ctas, bad);
  // dgrad: gy [N,H,W,Cout] -> dx [N,H,W,Cin] with the same filter
  if (Cout % 64 || Cin % 64) return;
  Mat gy(N * H * W, Cout);
  std::vector<uint16_t> dv(size_t(N) * H * W * Cin + 16, 0xdead);
  uint16_t* dx = dv.data();
  while (reinterpret_cast<uintptr_t>(dx) & 15) dx++;
  e = setup_conv(gy.ptr(), w.ptr(), nullptr, dx, N, H, W, Cout, Cin, 0, 1, &err, sms, &cp);
  CHECK(e == nullptr, "conv dgrad setup: %s", e ? e : "");
  if (e) return;
  if (cp.plan.bn == 64) run_conv_kernel<64, true>(cp, HostOut{});
  else if (cp.plan.bn == 128) run_conv_kernel<128, true>(cp, HostOut{});
  else run_conv_kernel<256, true>(cp, HostOut{});
  bad = 0;
  for (int n = 0; n < N; n++)
    for (int h = 0; h < H; h++)
      for (int ww = 0; ww < W; ww++)
        for (int ci = 0; ci < Cin; ci++) {
          double r = 0;
          for (int kh = 0; kh < 3; kh++)
            for (int kw = 0; kw < 3; kw++) {
              const int ho = h - kh + 1, wo = ww - kw + 1;      // the output pixel that read x[h, w] through tap (kh, kw)
              if (ho < 0 || ho >= H || wo < 0 || wo >= W) continue;
              for (int co = 0; co < Cout; co++) r += double(gy.at((n * H + ho) * W + wo, co)) * w.at(co, (kh * 3 + kw) * Cin + ci);
            }
          if (!close(bf16_to_f32(dx[(size_t(n * H + h) * W + ww) * Cin + ci]), r)) bad++;
        }
  CHECK(bad == 0, "conv dgrad N=%d %dx%d %d->%d (bn %d): %d wrong", N, H, W, Cin, Cout, cp.plan.bn, bad);
}

// ---- convolution weight gradient: both operands 4-D boxes of 64 pixels, MN-major; split over pixel blocks with the fix-up --
template <int BN>
static void run_wgrad_kernel(const WgradProblem& wp, const HostOut& out) {
  const TcArgs& args = wp.args;
  const BnetTcPlan& p = wp.plan;
  std::vector<uint16_t> stage_a(kABytes / 2), stage_b(BN * kBK);
  std::vector<float> accum(size_t(kBM) * BN);
  CHECK(args.conv.bw * args.conv.bh * args.conv.bn == 64, "wgrad patch %d x %d x %d", args.conv.bw, args.conv.bh, args.conv.bn);
  CHECK(wp.gy_map.bw * wp.gy_map.bh * wp.gy_map.bn == 64 && wp.x_map.bw * wp.x_map.bh * wp.x_map.bn == 64, "wgrad boxes");
  int* counters = args.fix_counters;
  float* ws = static_cast<float*>(args.outs[0]);
  for (int z = 0; z < p.grid_z; z++) {
    const int kb_begin = z * args.k_per_split;
    const int kb_end = kb_begin + args.k_per_split < args.k_blocks ? kb_begin + args.k_per_split : args.k_blocks;
    CHECK(kb_end > kb_begin, "empty pixel slice %d", z);
    for (int cta = 0; cta < p.ctas; cta++)
      for (int t = cta; t < args.n_tiles; t += p.ctas) {
        const TileCoord tc = tile_coord<BN, false>(args, t);
        std::fill(accum.begin(), accum.end(), 0.f);
        for (int kb = kb_begin; kb < kb_end; kb++) {
          std::fill(stage_a.begin(), stage_a.end(), uint16_t(0x7fc0));
          std::fill(stage_b.begin(), stage_b.end(), uint16_t(0x7fc0));
          int bytes = 0;
          wgrad_stage_loads<BN>(args, tc, kb,
              [&](int offset, int c0, int c1, int c2, int c3) { tma_box4(wp.gy_map, c0, c1, c2, c3, stage_a.data() + offset / 2); bytes += kAtomBytes; },
              [&](int offset, int c0, int c1, int c2, int c3) { tma_box4(wp.x_map, c0, c1, c2, c3, stage_b.data() + offset / 2); bytes += kAtomBytes; });
          CHECK(bytes == kABytes + BN * kBK * 2, "wgrad expect_tx bytes %d", bytes);
          for (int i = 0; i < kBM; i++)
            for (int j = 0; j < BN; j++) {
              float s = 0.f;
              for (int k = 0; k < kBK; k++) s += stage_at(stage_a.data(), true, i, k) * stage_at(stage_b.data(), true, j, k);
              accum[size_t(i) * BN + j] += s;
            }
        }
        // the epilogue of the reduce instantiation: fp32 adds into the workspace ...
        for (int r = 0; r < kBM; r++)
          for (int c = 0; c < BN / 16; c++) {
            float acc[16];
            for (int u = 0; u < 16; u++) acc[u] = accum[size_t(r) * BN + c * 16 + u];
            epilogue_chunk<false, true>(args, tc.a_row0 + r, tc.b_row0 + c * 16, acc, false, out);
          }
        // ... and the fix-up: the slice that arrives last at the tile reads the sums back, writes bf16, re-zeroes what it read
        if (args.fix_out != nullptr && ++counters[t] == p.grid_z) {
          TcArgs fa = args;
          fa.outs[0] = args.fix_out;
          fa.ldo = args.fix_ldo;
          for (int r = 0; r < kBM; r++) {
            const int i_glob = tc.a_row0 + r;
            if (i_glob >= args.rows_a) continue;
            for (int c = 0; c < BN / 16; c++) {
              const int j0 = tc.b_row0 + c * 16;
              if (j0 >= args.rows_b) break;
              float acc[16];
              for (int u = 0; u < 16; u++) {
                acc[u] = 0.f;
                if (j0 + u < args.rows_b) {
                  float* q = ws + size_t(i_glob) * args.ldo + j0 + u;
                  acc[u] = *q;
                  *q = 0.f;
                }
              }
              epilogue_chunk<false, false>(fa, i_glob, j0, acc, false, out);
            }
          }
          counters[t] = 0;
        }
      }
  }
}

static void conv_wgrad(int N, int H, int W, int Cin, int Cout, int sms, int splits, int force_bn = 0, int fixup = 1) {
  Mat gy(N * H * W, Cout), x(N * H * W, Cin);
  const int cols = 9 * Cin;
  std::vector<float> ws(size_t(Cout) * cols, 0.f);
  std::vector<int> counters(wgrad_max_tiles(Cin, Cout), 0);
  std::vector<uint16_t> dv(size_t(Cout) * cols + 16, 0xdead);
  uint16_t* dw = dv.data();
  while (reinterpret_cast<uintptr_t>(dw) & 15) dw++;
  int err = 0;
  WgradProblem wp;
  const char* e = setup_conv_wgrad(gy.ptr(), x.ptr(), ws.data(), dw, counters.data(), N, H, W, Cin, Cout, splits, &err, sms, &wp, force_bn, fixup);
  CHECK(e == nullptr, "wgrad setup: %s", e ? e : "");
  if (e) return;
  CHECK(force_bn == 0 || wp.plan.bn == force_bn, "forced tile width %d, plan has %d", force_bn, wp.plan.bn);
  CHECK(wp.args.n_tiles <= (int)counters.size(), "wgrad_max_tiles %zu < %d tiles", counters.size(), wp.args.n_tiles);
  CHECK((long long)wp.plan.ctas * wp.plan.grid_z <= (sms > wp.plan.grid_z ? sms : wp.plan.grid_z) || wp.plan.ctas == 1, "wgrad launches %d x %d CTAs on %d SMs",
        wp.plan.ctas, wp.plan.grid_z, sms);
  if (wp.plan.bn == 128) run_wgrad_kernel<128>(wp, HostOut{});
  else run_wgrad_kernel<256>(wp, HostOut{});
  if (!fixup)            // what the caller does in that mode: convert the sums, clear the workspace
    for (size_t i = 0; i < ws.size(); i++) { dw[i] = f32_to_bf16(ws[i]); ws[i] = 0.f; }
  int bad = 0;
  for (int co = 0; co < Cout; co++)
    for (int kh = 0; kh < 3; kh++)
      for (int kw = 0; kw < 3; kw++)
        for (int ci = 0; ci < Cin; ci++) {
          double r = 0;
          for (int n = 0; n < N; n++)
            for (int h = 0; h < H; h++)
              for (int w2 = 0; w2 < W; w2++) {
                const int hi = h + kh - 1, wi = w2 + kw - 1;          // the input pixel output (h, w) read through tap (kh, kw)
                if (hi < 0 || hi >= H || wi < 0 || wi >= W) continue;
                r += double(gy.at((n * H + h) * W + w2, co)) * x.at((n * H + hi) * W + wi, ci);
              }
          if (!close(bf16_to_f32(dw[size_t(co) * cols + (kh * 3 + kw) * Cin + ci]), r)) bad++;
        }
  if (getenv("TC_EMU_VERBOSE"))
    printf("  wgrad N=%d %dx%d %d->%d: patch %dx%dx%d, %d pixel blocks in %d slices, %d tiles of 128x%d on %d CTAs per slice, %d wrong\n", N, H, W,
           Cin, Cout, wp.args.conv.bw, wp.args.conv.bh, wp.args.conv.bn, wp.plan.k_blocks, wp.plan.grid_z, wp.args.n_tiles, wp.plan.bn,
           wp.plan.ctas, bad);
  int dirty = 0;
  for (float v : ws) dirty += v != 0.f;
  for (int c : counters) dirty += c != 0;
  CHECK(bad == 0 && dirty == 0, "conv wgrad N=%d %dx%d %d->%d (patch %dx%dx%d bn %d tiles %d slices %d ctas %d): %d wrong, %d scratch words left dirty",
        N, H, W, Cin, Cout, wp.args.conv.bw, wp.args.conv.bh, wp.args.conv.bn, wp.plan.bn, wp.args.n_tiles, wp.plan.grid_z, wp.plan.ctas, bad, dirty);
}

int main() {
  // filter gradients: exact and ragged 64-pixel patches, Cout below / above one lane tile, tiles that straddle taps (Cin = 64
  // with 128 columns), columns past 9 * Cin (Cin = 128 with 256-column tiles), one slice / many slices / persistent CTAs
  conv_wgrad(2, 8, 8, 64, 64, 132, 0);
  conv_wgrad(3, 7, 7, 64, 128, 4, 0);
  conv_wgrad(1, 14, 14, 128, 64, 132, 3);
  conv_wgrad(5, 4, 4, 64, 192, 2, 1);
  conv_wgrad(2, 6, 10, 128, 256, 7, 0);
  conv_wgrad(1, 5, 3, 256, 128, 132, 0);
  conv_wgrad(2, 6, 10, 128, 256, 7, 0, 128);         // the self-check's fallback: 128-column tiles for every layer
  conv_wgrad(1, 5, 3, 256, 128, 132, 2, 128);
  conv_wgrad(3, 7, 7, 64, 128, 4, 0, 0, 0);          // ... and without the in-kernel finish (the caller converts the workspace)
  conv_wgrad(2, 6, 10, 128, 256, 7, 2, 128, 0);
  // forward / input gradient: exact patches, ragged patches (7x7, 14x14 with odd batch), several images per patch, persistent CTAs
  conv(2, 8, 16, 64, 64, true, 132);
  conv(3, 7, 7, 64, 128, false, 3);
  conv(1, 14, 14, 128, 64, true, 2);
  conv(5, 4, 4, 64, 72, true, 132);
  conv(2, 10, 6, 64, 320, false, 1);
  // forward: both orientations, ragged extents, row pitches, one tile per CTA and persistent (few "SMs")
  forward(32, 256, 512, true, true, 132, 0);
  forward(48, 200, 264, true, false, 132, 16);
  forward(1, 8, 8, false, false, 132, 0);
  forward(64, 130, 72, true, true, 2, 0);
  forward(130, 136, 72, true, false, 132, 8);
  forward(257, 129, 200, false, true, 3, 0);
  forward(300, 520, 136, true, true, 4, 0);
  forward(256, 512, 64, true, false, 2, 0);           // 128 x 256 tiles (2 x 2 of them >= 2 SMs)
  // GEMM + all-reduce: per-peer adds, multicast, split-K, bias once
  reduce(32, 136, 264, 3, false, 1, 0, true);
  reduce(32, 136, 520, 2, false, 4, 0, true);
  reduce(130, 200, 264, 3, false, 2, 0, false);
  reduce(40, 72, 136, 1, true, 1, 0, true);
  reduce(256, 136, 200, 1, true, 3, 0, true);
  // GEMM + reduce-scatter
  reduce(96, 136, 264, 0, false, 1, 3, true);
  reduce(512, 72, 136, 0, false, 2, 4, false);
  reduce(48, 200, 72, 0, false, 1, 2, true);
  // all-gather + GEMM
  gather(2, 128, 136, 200);
  gather(3, 256, 72, 72);
  // backward GEMMs: MN-major operands, both orientations of dX
  backward(32, 136, 264);
  backward(64, 72, 136);
  backward(130, 200, 72);
  backward(256, 320, 192);
  backward(40, 64, 128);
  // randomised extents (multiples of 8 where TMA needs them), every mode
  for (int it = 0; it < 40; it++) {
    auto r = [&](int lo, int hi) { g_rng = g_rng * 1664525u + 1013904223u; return lo + int((g_rng >> 8) % uint32_t(hi - lo + 1)); };
    const int M = r(1, 300), N = r(1, 40) * 8, K = r(1, 40) * 8, sms = r(1, 6);
    forward(M, N, K, r(0, 1), r(0, 1), sms, r(0, 1) * 8);
    if (it % 4 == 0) reduce(M, N, K, r(1, 4), false, r(1, 5), 0, r(0, 1));
    if (it % 4 == 1) reduce(M, N, K, 1, true, r(1, 3), 0, r(0, 1));
    if (it % 4 == 2) { const int ranks = r(2, 4); reduce(M * ranks, N, K, 0, false, r(1, 3), ranks, r(0, 1)); }
    if (it % 4 == 3) backward(r(1, 40) * 8, N, K);
    if (it % 8 == 5) gather(r(2, 4), 128 * r(1, 2), N, K);
  }
  printf("tc_emu_test: %s (%d failures)\n", g_failures ? "FAILED" : "passed", g_failures);
  return g_failures ? 1 : 0;
}
