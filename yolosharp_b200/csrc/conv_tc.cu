// wgmma implicit-GEMM convolution for sm_90a (fp16 NHWC activations, fp32 accumulate in registers).
//
// Computes the reference's Conv block (Modules/Convs.cs:36-56: Conv2d -> BatchNorm2d -> SiLU, BN
// folded into weights/bias at load) and the Bottleneck shortcut (Block.cs:606) as ONE kernel:
//
//   GEMM view   M = output pixels (tile = 128 rows = a BW x BH rectangle of one image, or 128
//               consecutive pixels of the flattened batch for 1x1 convs)
//               N = Cout (tile = n_tile <= 256), K = taps * Cin walked tap-major in slabs of BK
//   A operand   per (tap, channel slab): one 4-D TMA box {BK, BW, BH, 1} of the NHWC input view at
//               (w0*s + kw - pad, h0*s + kh - pad); out-of-bounds rows/cols are zero-filled by TMA
//               (= conv zero padding), stride-2 convs use the tensor map's traversal stride
//   B operand   weights [Cout][tap][Cin] fp16, 2-D TMA box {BK, n_tile}
//   swizzle     BK = 64/32/16 channels -> SWIZZLE_128B/64B/32B rows, identical in the TMA map and
//               the wgmma shared-memory descriptors
//   MMA         wgmma.mma_async m64nNk16 f16 -> f32: two consumer warpgroups, each owning 64 rows of the
//               tile and its n_tile accumulator columns in registers
//   epilogue    the same warpgroups: +bias -> SiLU -> +residual -> fp16 stores into the channel slice of
//               the (concat) output buffer
//   schedule    persistent CTAs (one or two per SM), warp-specialised: warps 0-7 = consumers, warp 8 = TMA
//               producer; smem rings of `stages` slabs the producer fills ahead of the consumers.
#include <cuda.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <utility>
#include <vector>

#include "common.cuh"
#include "tc_ptx.cuh"

namespace yb {

// Grid of a persistent launch of `total` tiles on at most `max_grid` CTAs, and the tiles per draw from the launch's
// counter: one atomic per ~quarter of a CTA's share (every atomic of the grid hits the same L2 address, so per-tile
// draws would serialise the 6400-tile layers)
static int tc_grid(int max_grid, int total, int* tile_batch) {
  const int grid = std::min(max_grid, total);
  *tile_batch = std::max(1, std::min(8, total / (4 * grid)));
  return grid;
}

enum TcMode { TC_TAP = 0, TC_HALO = 1, TC_S2P = 2 };

struct TcArgs {
  CUtensorMap tmA;
  const uint8_t* wpk;  // weights pre-packed as shared-memory slab images [n tile][tap][chunk][b_stride bytes]
  __half* out;
  const __half* res;
  const float* bias;
  int out_pitch, out_coff, res_pitch, res_coff;
  int Ho, Wo;            // output extent the tiles cover (flattened for 1x1: Ho = 1, Wo = B*H*W)
  int imgs;              // images the tiles iterate over (1 for flattened 1x1)
  TileGrid tg;
  int BW, BH;
  int n_tile, n_tiles;
  int ksz, stride, pad;
  int Cin, BK, chunks;   // chunks = Cin / BK
  int act;
  int mode;                       // TcMode
  int stages_a, stages_b;
  uint32_t a_bytes, b_bytes;      // TMA transaction bytes per A slab / B slab
  uint32_t a_stride, b_stride;    // smem bytes reserved per slab (1 KiB aligned)
  uint32_t sbo_a, sbo_b;          // wgmma stride-byte-offset between 8-row groups, >> 4
  uint32_t row_bytes;             // BK * 2
  uint32_t layout_a, layout_b;    // wgmma layout type: 1 = SW128, 2 = SW64, 3 = SW32
  int b_resident;                 // all weight slabs stay in smem for the CTA's lifetime
  int ksteps;
  // fused head decode (EpiDecode)
  int epi_mode, dA, dCtot, da0, dch0, dWl, dHW;
  float dstride;
  float* pred;
  uint64_t m_bw;   // fdiv magic of BW
  int* tile_ctr;   // tile queue: global counter of this launch (nullptr = round-robin order)
  int tile_batch;  // consecutive tiles drawn per atomicAdd (one counter address serves the whole grid)
  long long* dbg;  // optional timeline buffer (tools/exp_timeline.py); nullptr in production
  // folded 1x1 (tc_fold, conv_tc_kernel<NT16, N2_16 > 0>): this conv's activations never leave registers; the next conv, a
  // 1x1, multiplies them with its weights and runs the epilogue described above (out / act / epi_mode are the 1x1's)
  const uint8_t* w2;  // the 1x1's packed weight slabs (pack_weights_kernel, taps = 1), resident in smem at w2_off
  const float* bias2;
  uint32_t w2_off, w2_bytes, b2_stride, sbo_b2, layout_b2;
  int BK2, n2, act1;  // the 1x1's slab width and Cout; this conv's activation
};

struct TcConvPlan {
  TcArgs args;
  ConvParams p;
  bool flat;   // 1x1 stride-1 conv on the flattened pixel dimension
  int occ;     // CTAs per SM this plan is sized for
  bool small;  // <= 2 tiles per CTA
  size_t smem;
  int grid;
  uint8_t* wpk = nullptr;  // device, owned: packed weight slabs
  void (*kernel)(TcArgs) = nullptr;  // conv_tc_kernel<n_tile / 16> (<n_tile / 16, fold16> for a folded 1x1)
  int fold16 = 0;                    // folded 1x1 (tc_fold_plan_create): its column pass width / 16
};
// a plan under construction: every refusal frees its packed weights
struct TcPlanDestroy { void operator()(TcConvPlan* plan) const { tc_conv_plan_destroy(plan); } };
using TcPlanPtr = std::unique_ptr<TcConvPlan, TcPlanDestroy>;

// x*sigmoid(x) = h + h*tanh(h), h = x/2: one MUFU op instead of two (ex2 + rcp)
__device__ __forceinline__ float silu_tanh(float v) {
  const float h = 0.5f * v;
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(h));
  return fmaf(h, t, h);
}

__device__ __forceinline__ uint32_t pack_h2(float x, float y) {
  const __half2 h = __floats2half2_rn(x, y);
  return *reinterpret_cast<const uint32_t*>(&h);
}

// Accumulator pair acc[0..1] (columns c, c + 1) + bias[c..c + 1] -> SiLU when `silu`: the rounding points every fp16
// epilogue of this file starts with (fp32 sum + bias, then the activation); the caller adds a residual and rounds to fp16.
__device__ __forceinline__ float2 bias_act(const float* acc, const float* bias, bool silu) {
  const float2 b = *reinterpret_cast<const float2*>(bias);
  float2 f = make_float2(acc[0] + b.x, acc[1] + b.y);
  if (silu) { f.x = silu_tanh(f.x); f.y = silu_tanh(f.y); }
  return f;
}

// Descriptor start shift (16-byte units) of 3x3 tap t inside a staged tile of `pitch`-pixel rows, row16 units per pixel
__device__ __forceinline__ uint32_t tap_shift(int t, int pitch, uint32_t row16) {
  return (uint32_t)((t / 3) * pitch + t % 3) * row16;
}

constexpr int TC_CONSUMERS = 256;                // warps 0-7: two warpgroups, rows 0-63 / 64-127 of every tile
constexpr int TC_THREADS = TC_CONSUMERS + 32;    // warp 8: TMA producer
constexpr int TC_CONSUMER_WARPS = TC_CONSUMERS / 32;
constexpr int TC_MAX_COUT = 1024;
constexpr int TC_MAX_STAGES = 12;
constexpr int HALO_BW = 8, HALO_BH = 16;  // output rectangle of a halo tile (128 rows)

// ------------------------------------------------------------------------------------------
// Dynamic tile scheduler.  The producer thread draws tile indices from a global counter (first tile =
// blockIdx.x, then gridDim.x + atomicAdd) and publishes them in a small shared-memory queue that the consumer
// warpgroups follow.  CTAs that start late - SMs held by a concurrent kernel (NMS of the previous batch, a sibling
// head branch) - simply take fewer tiles instead of delaying the whole grid with a fixed share.  The queue cannot
// wrap onto unread entries: every tile takes at least one ring slot, so the producer is at most stages_a (< 32)
// tiles ahead of the consumers.
// ------------------------------------------------------------------------------------------
constexpr int TQ = 32;
__device__ __forceinline__ void tq_publish(int* s_tile, volatile int* s_head, int li, int tile) {
  s_tile[li & (TQ - 1)] = tile;
  __threadfence_block();
  *s_head = li + 1;
}
__device__ __forceinline__ int tq_get(const int* s_tile, const volatile int* s_head, int li) {
  const long long t0 = clock64();
  while (*s_head <= li)
    if (clock64() - t0 > 4000000000ll) __trap();
  __threadfence_block();
  return reinterpret_cast<const volatile int*>(s_tile)[li & (TQ - 1)];
}
// The producer's tile sequence: blockIdx.x first, then batches of `batch` consecutive tiles from the launch's counter,
// each drawn one batch ahead so that the atomic's latency never sits on the load path (ctr == nullptr: round-robin).
struct TileDraw {
  int tile, nxt, left, batch, total;
  int* ctr;
  __device__ __forceinline__ TileDraw(int* c, int b, int tot)
      : tile((int)blockIdx.x), nxt(tot), left(1), batch(b), total(tot), ctr(c) {
    if (ctr && tile < total) nxt = (int)gridDim.x + atomicAdd(ctr, batch);
  }
  __device__ __forceinline__ void advance() {
    if (!ctr) { tile += gridDim.x; return; }
    if (--left > 0) { tile++; return; }
    tile = nxt;
    left = batch;
    if (tile < total) nxt = (int)gridDim.x + atomicAdd(ctr, batch);
  }
};

// ------------------------------------------------------------------------------------------
// Main loop of one tile for one consumer warpgroup (its 64 rows of the 128-row tile, all n_tile columns).
// Every K step is one wgmma commit group; after issuing group g the warpgroup waits for group g-1 and frees the ring
// slots g-1 read (one arrive per warp: the empty barriers count 8), so the tensor pipe always has the next group
// queued while a slot is handed back to the producer.
//   TC_TAP  - one 128-row A slab per (tap, channel slab)
//   TC_HALO - one (BH+2)x(BW+2)-pixel halo tile per channel slab; the 9 taps of a 3x3 stride-1 conv are issued from
//             the SAME bytes with the descriptor start shifted by (kh*(BW+2)+kw) rows and SBO = (BW+2) rows (the
//             swizzle follows absolute address bits, tc_ptx.cuh) -> 180 TMA rows per slab instead of 9 x 128
//   TC_S2P  - stride-2 pair rows, the same idea with (input row, pair, half) shifts
// B: one [n_tile x BK] weight slab per (tap, channel slab), streamed through its own ring or all resident.
// ------------------------------------------------------------------------------------------
template <int NT16, int KK>
__device__ __forceinline__ void tc_mainloop(const TcArgs& a, float* acc, int wg, uint32_t smemA, uint32_t smemB, uint32_t fullA,
                                            uint32_t emptyA, uint32_t fullB, uint32_t emptyB, int& sa, uint32_t& pa, int& sb,
                                            uint32_t& pb) {
  const bool resident = a.b_resident != 0, halo = a.mode != TC_TAP, s2p = a.mode == TC_S2P;
  const uint32_t a_hi = wg_desc_hi(a.sbo_a, a.layout_a), b_hi = wg_desc_hi(a.sbo_b, a.layout_b);
  const uint32_t a_stride16 = a.a_stride >> 4, b_stride16 = a.b_stride >> 4;
  const uint32_t a_lo0 = wg_desc_lo(smemA) + (uint32_t)wg * 8 * a.sbo_a;  // rows 64 * wg.. = 8 groups of 8 rows further
  const uint32_t b_lo0 = wg_desc_lo(smemB);
  constexpr uint32_t ROW16 = KK * 2;  // bytes per operand row / 16
  const int ra = a.stages_a, rb = a.stages_b;
  const bool leader = (threadIdx.x & 31) == 0;
  uint32_t pend0 = 0, pend1 = 0;  // slots read by the previous commit group
  uint32_t scale = 0;
  auto step = [&](uint32_t a_lo, uint32_t b_lo, uint32_t relA, uint32_t relB) {
    wg_fence();
#pragma unroll
    for (int k = 0; k < KK; k++) {  // +32 B per K=16 step inside the swizzled row
      wg_mma_n<NT16, false>(acc, a_lo + 2 * k, a_hi, b_lo + 2 * k, b_hi, ROW16, scale);
      scale = 1;
    }
    wg_commit();
    wg_wait<1>();
    __syncwarp();
    if (leader) {
      if (pend0) mbar_arrive(pend0);
      if (pend1) mbar_arrive(pend1);
    }
    pend0 = relA;
    pend1 = relB;
  };
  if (halo) {
    for (int ch = 0; ch < a.chunks; ch++) {
      mbar_wait(fullA + 8 * sa, pa);
      const uint32_t a_lo = a_lo0 + sa * a_stride16;
      const uint32_t slotA = emptyA + 8 * sa;
      ring_next(sa, pa, ra);
#pragma unroll
      for (int t = 0; t < 9; t++) {
        // row shift of tap t inside the staged input tile (compile-time constants after unrolling):
        //   halo : (kh * (BW+2) + kw) pixel rows
        //   s2p  : pair rows (input pixels 2q, 2q+1), the tile starts at pair w0-1: kw = 0 is the second half
        //          of pair j, kw = 1 / 2 the two halves of pair j+1; kh advances one input row = (BW+1) pairs
        const uint32_t TAP_HALO = tap_shift(t, HALO_BW + 2, ROW16);
        const uint32_t TAP_S2P = (uint32_t)((t / 3) * (HALO_BW + 1) + (t % 3 != 0 ? 1 : 0)) * 2 * ROW16 +
                                 (t % 3 != 1 ? ROW16 : 0);
        const uint32_t tap16 = s2p ? TAP_S2P : TAP_HALO;
        uint32_t b_lo, relB = 0;
        if (resident) {
          b_lo = b_lo0 + (t * a.chunks + ch) * b_stride16;
        } else {
          mbar_wait(fullB + 8 * sb, pb);
          b_lo = b_lo0 + sb * b_stride16;
          relB = emptyB + 8 * sb;
          ring_next(sb, pb, rb);
        }
        step(a_lo + tap16, b_lo, t == 8 ? slotA : 0u, relB);  // halo tile free once its 9 taps retired
      }
    }
  } else {
    for (int ks = 0; ks < a.ksteps; ks++) {
      mbar_wait(fullA + 8 * sa, pa);
      const uint32_t a_lo = a_lo0 + sa * a_stride16;
      const uint32_t relA = emptyA + 8 * sa;
      ring_next(sa, pa, ra);
      uint32_t b_lo, relB = 0;
      if (resident) {
        b_lo = b_lo0 + ks * b_stride16;
      } else {
        mbar_wait(fullB + 8 * sb, pb);
        b_lo = b_lo0 + sb * b_stride16;
        relB = emptyB + 8 * sb;
        ring_next(sb, pb, rb);
      }
      step(a_lo, b_lo, relA, relB);
    }
  }
  wg_wait<0>();
  __syncwarp();
  if (leader) {
    if (pend0) mbar_arrive(pend0);
    if (pend1) mbar_arrive(pend1);
  }
  wg_fence_acc<NT16 * 8>(acc);
}

// Epilogue of one tile from the accumulator registers: +bias -> SiLU -> +residual -> fp16 into the channel slice of
// the (concat) output buffer, or the fused Detect tail (DFL box decode / class scores into the prediction tensor).
template <int NT16>
__device__ __forceinline__ void tc_epilogue(const TcArgs& a, const float* acc, const float* bias, int n0, int img, int th,
                                            int tw, int wg) {
  const int t4 = threadIdx.x & 3;
  size_t pix[2];
  int ho[2], wo[2];
  bool valid[2];
#pragma unroll
  for (int h = 0; h < 2; h++) {
    const int row = acc_row(wg, h);
    const int hl = fdiv(row, a.m_bw), wl = row - hl * a.BW;
    ho[h] = th * a.BH + hl;
    wo[h] = tw * a.BW + wl;
    valid[h] = hl < a.BH && ho[h] < a.Ho && wo[h] < a.Wo;
    pix[h] = ((size_t)img * a.Ho + ho[h]) * a.Wo + wo[h];
  }
  if (a.epi_mode != EPI_STORE) {
    // fused Detect tail: row h of this thread is anchor i of image n - pixel wo[h] of the whole batch for a flattened
    // tile, (ho, wo) of image img for a rectangular one (a 1x1 folded into a 3x3 producer)
    const bool flat1 = a.imgs == 1 && a.Ho == 1;
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int n = flat1 ? (valid[h] ? wo[h] / a.dHW : 0) : img;
      const int i = flat1 ? wo[h] - n * a.dHW : ho[h] * a.dWl + wo[h];
      float* po = a.pred + (size_t)n * a.dCtot * a.dA + a.da0 + i;
      if (a.epi_mode == EPI_DFL_BOX) {
        if constexpr (NT16 == 4) {  // the plans refuse a DFL epilogue whose n_tile / pass is not 64 = 4 sides x 16 bins
          // DFL (Block.cs:44): softmax over the 16 bins of each side, expectation with weights 0..15; then
          // dist2bbox(xywh) * stride (Tal.cs:338-356, Head.cs:221).  A quad of lanes holds the 16 bins of a side.
          float d[4];
#pragma unroll
          for (int sd = 0; sd < 4; sd++) {
            const int b0 = 2 * t4;
            float f[4];
            f[0] = acc[4 * (2 * sd) + 2 * h] + bias[16 * sd + b0];
            f[1] = acc[4 * (2 * sd) + 2 * h + 1] + bias[16 * sd + b0 + 1];
            f[2] = acc[4 * (2 * sd + 1) + 2 * h] + bias[16 * sd + 8 + b0];
            f[3] = acc[4 * (2 * sd + 1) + 2 * h + 1] + bias[16 * sd + 9 + b0];
            float mx = fmaxf(fmaxf(f[0], f[1]), fmaxf(f[2], f[3]));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            const float bin[4] = {(float)b0, (float)(b0 + 1), (float)(b0 + 8), (float)(b0 + 9)};
            float sum = 0.f, ex = 0.f;
#pragma unroll
            for (int j = 0; j < 4; j++) { const float e = __expf(f[j] - mx); sum += e; ex = fmaf(e, bin[j], ex); }
            sum += __shfl_xor_sync(0xffffffffu, sum, 1);
            ex += __shfl_xor_sync(0xffffffffu, ex, 1);
            sum += __shfl_xor_sync(0xffffffffu, sum, 2);
            ex += __shfl_xor_sync(0xffffffffu, ex, 2);
            d[sd] = __fdividef(ex, sum);
          }
          if (valid[h] && t4 == 0) {
            const int y = i / a.dWl, x = i - y * a.dWl;
            const float ax = (float)x + 0.5f, ay = (float)y + 0.5f;
            const float x1 = ax - d[0], y1 = ay - d[1], x2 = ax + d[2], y2 = ay + d[3];
            po[0] = (x1 + x2) * 0.5f * a.dstride;
            po[(size_t)a.dA] = (y1 + y2) * 0.5f * a.dstride;
            po[(size_t)2 * a.dA] = (x2 - x1) * a.dstride;
            po[(size_t)3 * a.dA] = (y2 - y1) * a.dstride;
          }
        }
      } else if (valid[h]) {
#pragma unroll
        for (int J = 0; J < NT16 * 2; J++)
#pragma unroll
          for (int e = 0; e < 2; e++) {
            const int c = 8 * J + 2 * t4 + e;
            float f = acc[4 * J + 2 * h + e] + bias[c];
            if (a.epi_mode == EPI_SIGMOID) f = __fdividef(1.0f, 1.0f + __expf(-f));
            po[(size_t)(a.dch0 + n0 + c) * a.dA] = f;
          }
      }
    }
    return;
  }
  const bool use_res = a.res != nullptr;
#pragma unroll
  for (int h = 0; h < 2; h++) {
    if (!valid[h]) continue;
    __half* orow = a.out + pix[h] * a.out_pitch + a.out_coff + n0;
    const __half* rrow = use_res ? a.res + pix[h] * a.res_pitch + a.res_coff + n0 : nullptr;
#pragma unroll
    for (int J = 0; J < NT16 * 2; J++) {
      const int c = 8 * J + 2 * t4;
      float2 f = bias_act(acc + 4 * J + 2 * h, bias + c, a.act == ACT_SILU);
      if (use_res) {
        // L2-only load: every residual element is read exactly once, so an L1 copy of its line would never be reused
        const unsigned int rb = __ldcg(reinterpret_cast<const unsigned int*>(rrow + c));
        const float2 x = __half22float2(*reinterpret_cast<const __half2*>(&rb));
        f.x += x.x; f.y += x.y;
      }
      *reinterpret_cast<__half2*>(orow + c) = __floats2half2_rn(f.x, f.y);
    }
  }
}

// Folded 1x1 of one tile for one consumer warpgroup.  The tile's accumulator (this conv, NT16 * 16 channels) goes
// through the unfused store path's +bias -> activation -> fp16 rounding, but into registers: f16 pairs in the A-fragment
// layout, 16 channels per k16 step (tc_ptx.cuh, wgmma_f16_rs).  The 1x1 then runs in passes of F16 * 16 output
// columns against its resident weight slabs, each pass followed by the 1x1's epilogue.  Its k16 steps are those of the
// unfused 1x1 launch, in the same channel order on the same fp16 operands; that launch's extra steps over a ragged
// last slab multiply zeros.  The passes are unrolled, so the fragments die with the last pass's MMAs, before its epilogue.
__host__ __device__ constexpr int tc_fold_pass16(int n2_16) {  // column pass width / 16 (0: no pass width fits)
  return n2_16 <= 5 ? n2_16 : (n2_16 % 4 == 0 ? 4 : (n2_16 % 5 == 0 ? 5 : 0));
}

template <int NT16, int N2_16, int KK2>
__device__ __forceinline__ void tc_fold(const TcArgs& a, const float* acc, const float* bias1, const float* bias2,
                                        uint32_t smemW2, int img, int th, int tw, int wg) {
  constexpr int F16 = tc_fold_pass16(N2_16);
  static_assert(F16 > 0 && N2_16 % F16 == 0, "the 1x1's Cout must split into column passes of <= 80");
  const int t4 = threadIdx.x & 3;
  uint32_t fr[NT16 * 4];
#pragma unroll
  for (int J = 0; J < NT16 * 2; J++)
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const float2 f = bias_act(acc + 4 * J + 2 * h, bias1 + 8 * J + 2 * t4, a.act1 == ACT_SILU);
      fr[2 * J + h] = pack_h2(f.x, f.y);  // k step J / 2: fr[4 (J / 2) + 2 (J % 2) + h]
    }
  constexpr uint32_t ROW16 = KK2 * 2;  // bytes per weight row / 16
  const uint32_t b_hi = wg_desc_hi(a.sbo_b2, a.layout_b2);
  const uint32_t b_lo0 = wg_desc_lo(smemW2), b_slab16 = a.b2_stride >> 4;
#pragma unroll
  for (int c0 = 0; c0 < 16 * N2_16; c0 += 16 * F16) {
    float acc2[F16 * 8];
    wg_fence();
#pragma unroll
    for (int kk = 0; kk < NT16; kk++)
      wg_mma_rs_n<F16>(acc2, fr + 4 * kk, b_lo0 + (kk / KK2) * b_slab16 + (uint32_t)c0 * ROW16 + 2 * (kk % KK2), b_hi, ROW16,
                       kk > 0 ? 1u : 0u);
    wg_commit();
    wg_wait<0>();
    wg_fence_acc<F16 * 8>(acc2);
    tc_epilogue<F16>(a, acc2, bias2 + c0, c0, img, th, tw, wg);
  }
}

constexpr int TC_FOLD_BIAS = 256;  // s_bias offset of the folded 1x1's bias (this conv has one N tile of <= 256)

// CTAs per SM an instantiation's register bound allows without spills (ptxas -v): two leave 96 registers per thread,
// room for 64 accumulator columns, or a fold whose two accumulators add up to that (32 -> 32).  A 64 -> 64 fold wants
// ~150 registers and runs one CTA per SM.
__host__ __device__ constexpr int tc_ctas_per_sm(int nt16, int n2_16) { return nt16 <= 4 && nt16 + n2_16 <= 4 ? 2 : 1; }

// N2_16 > 0: a folded 1x1 of N2_16 * 16 output channels (tc_fold)
template <int NT16, int N2_16 = 0>
__global__ void __launch_bounds__(TC_THREADS, tc_ctas_per_sm(NT16, N2_16)) conv_tc_kernel(const __grid_constant__ TcArgs a) {
  extern __shared__ __align__(1024) uint8_t tc_smem[];
  __shared__ __align__(8) uint64_t bars[4 * TC_MAX_STAGES + 1];
  __shared__ int s_tile[TQ];
  __shared__ volatile int s_head;
  __shared__ __align__(16) float s_bias[TC_MAX_COUT];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < a.n_tile * a.n_tiles; i += blockDim.x) s_bias[i] = a.bias[i];  // constant data
  if constexpr (N2_16 > 0)
    for (int i = threadIdx.x; i < a.n2; i += blockDim.x) s_bias[TC_FOLD_BIAS + i] = a.bias2[i];
  // dynamic smem base rounded up to 1 KiB (SWIZZLE_128B atoms need it)
  const uint32_t smem0 = (smem_u32(tc_smem) + 1023u) & ~1023u;
  const uint32_t smemA = smem0;
  const uint32_t smemB = smem0 + a.stages_a * a.a_stride;
  const uint32_t fullA = smem_u32(&bars[0]);
  const uint32_t emptyA = smem_u32(&bars[TC_MAX_STAGES]);
  const uint32_t fullB = smem_u32(&bars[2 * TC_MAX_STAGES]);
  const uint32_t emptyB = smem_u32(&bars[3 * TC_MAX_STAGES]);
  const uint32_t bfull = smem_u32(&bars[4 * TC_MAX_STAGES]);

  // PDL: let the next kernel of the stream/graph start its prologue while this grid runs; it blocks in
  // its own pdl_wait() until this grid has completed and flushed.
  pdl_trigger();

  if (warp == TC_CONSUMER_WARPS && lane == 0) {
    s_head = 0;
    for (int s = 0; s < a.stages_a; s++) {
      mbar_init(fullA + 8 * s, 1);
      mbar_init(emptyA + 8 * s, TC_CONSUMER_WARPS);
    }
    for (int s = 0; s < a.stages_b; s++) {
      mbar_init(fullB + 8 * s, 1);
      mbar_init(emptyB + 8 * s, TC_CONSUMER_WARPS);
    }
    mbar_init(bfull, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  const int taps = a.ksz * a.ksz;

  if (warp == TC_CONSUMER_WARPS && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&a.tmA) : "memory");
    if (a.b_resident || N2_16 > 0) {
      // weights do not depend on the previous kernel: fetch them before the grid dependency resolves
      mbar_arrive_expect_tx(bfull, (a.b_resident ? a.b_bytes * a.ksteps : 0u) + (N2_16 > 0 ? a.w2_bytes : 0u));
      if (a.b_resident)
        for (int ks = 0; ks < a.ksteps; ks++)
          bulk_load_1d(smemB + ks * a.b_stride, a.wpk + (size_t)ks * a.b_stride, a.b_bytes, bfull);
      if (N2_16 > 0) bulk_load_1d(smem0 + a.w2_off, a.w2, a.w2_bytes, bfull);  // the folded 1x1's slabs, one copy
    }
  }
  // activations written by the previous kernel are visible only after this point
  pdl_wait();

  if (warp == TC_CONSUMER_WARPS) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      const int ra = a.stages_a, rb = a.b_resident ? 0 : a.stages_b;
      int sa = 0, sb = 0;
      uint32_t pa = 0, pb = 0;
      int li = 0;
      TileDraw td(a.tile_ctr, a.tile_batch, a.tg.total);
      for (; td.tile < a.tg.total; li++) {
        if (a.tile_ctr) tq_publish(s_tile, &s_head, li, td.tile);
        const TileCoord tc = tile_coord(a.tg, td.tile);
        const int wbase = tc.tw * a.BW * a.stride - a.pad;
        const int hbase = tc.th * a.BH * a.stride - a.pad;
        auto load_b = [&](int t, int ch) {
          mbar_wait(emptyB + 8 * sb, pb ^ 1);
          mbar_arrive_expect_tx(fullB + 8 * sb, a.b_bytes);
          bulk_load_1d(smemB + sb * a.b_stride, a.wpk + (size_t)((tc.nt * taps + t) * a.chunks + ch) * a.b_stride, a.b_bytes,
                       fullB + 8 * sb);
          ring_next(sb, pb, rb);
        };
        if (a.mode != TC_TAP) {
          for (int ch = 0; ch < a.chunks; ch++) {
            mbar_wait(emptyA + 8 * sa, pa ^ 1);
            mbar_arrive_expect_tx(fullA + 8 * sa, a.a_bytes);
            tma_load_4d(smemA + sa * a.a_stride, &a.tmA, fullA + 8 * sa, ch * a.BK, a.mode == TC_S2P ? tc.tw * a.BW - 1 : wbase,
                        hbase, tc.img);
            ring_next(sa, pa, ra);
            if (!a.b_resident)
              for (int t = 0; t < taps; t++) load_b(t, ch);
          }
        } else {
          for (int t = 0; t < taps; t++) {
            const int kh = a.ksz == 3 ? (t >= 6 ? 2 : (t >= 3 ? 1 : 0)) : 0, kw = t - kh * a.ksz;
            for (int ch = 0; ch < a.chunks; ch++) {
              mbar_wait(emptyA + 8 * sa, pa ^ 1);
              mbar_arrive_expect_tx(fullA + 8 * sa, a.a_bytes);
              tma_load_4d(smemA + sa * a.a_stride, &a.tmA, fullA + 8 * sa, ch * a.BK, wbase + kw, hbase + kh, tc.img);
              ring_next(sa, pa, ra);
              if (!a.b_resident) load_b(t, ch);
            }
          }
        }
        td.advance();
      }
      if (a.tile_ctr) tq_publish(s_tile, &s_head, li, -1);  // end mark
    }
  } else {
    // ===================== consumers: wgmma main loop + epilogue =====================
    const int wg = warp >> 2;
    int sa = 0, sb = 0;
    uint32_t pa = 0, pb = 0;
    if (a.b_resident || N2_16 > 0) mbar_wait(bfull, 0);
    const bool dbg_on = a.dbg && blockIdx.x == 0 && threadIdx.x == 0;
    for (int li = 0;; li++) {
      // without a counter (round-robin order) the consumers compute the producer's sequence themselves; sending it
      // through the queue as well costs up to 4 registers and a spill in some instantiations (ptxas -v, CUDA 12.9)
      const int tile = a.tile_ctr ? tq_get(s_tile, &s_head, li) : (int)blockIdx.x + li * (int)gridDim.x;
      if (tile < 0 || tile >= a.tg.total) break;
      if (dbg_on && li < 16) a.dbg[li * 8 + 0] = clock64();
      float acc[NT16 * 8];
      switch (a.BK) {
        case 64: tc_mainloop<NT16, 4>(a, acc, wg, smemA, smemB, fullA, emptyA, fullB, emptyB, sa, pa, sb, pb); break;
        case 32: tc_mainloop<NT16, 2>(a, acc, wg, smemA, smemB, fullA, emptyA, fullB, emptyB, sa, pa, sb, pb); break;
        default: tc_mainloop<NT16, 1>(a, acc, wg, smemA, smemB, fullA, emptyA, fullB, emptyB, sa, pa, sb, pb); break;
      }
      if (dbg_on && li < 16) a.dbg[li * 8 + 3] = clock64();
      const TileCoord tc = tile_coord(a.tg, tile);
      if constexpr (N2_16 > 0) {  // one N tile: n0 = 0
        switch (a.BK2) {
          case 64: tc_fold<NT16, N2_16, 4>(a, acc, s_bias, s_bias + TC_FOLD_BIAS, smem0 + a.w2_off, tc.img, tc.th, tc.tw, wg); break;
          case 32: tc_fold<NT16, N2_16, 2>(a, acc, s_bias, s_bias + TC_FOLD_BIAS, smem0 + a.w2_off, tc.img, tc.th, tc.tw, wg); break;
          default: tc_fold<NT16, N2_16, 1>(a, acc, s_bias, s_bias + TC_FOLD_BIAS, smem0 + a.w2_off, tc.img, tc.th, tc.tw, wg); break;
        }
      } else {
        const int n0 = tc.nt * a.n_tile;
        tc_epilogue<NT16>(a, acc, s_bias + n0, n0, tc.img, tc.th, tc.tw, wg);
      }
      if (dbg_on && li < 16) a.dbg[li * 8 + 6] = clock64();
    }
  }
}

// One-time weight packing: w [Cout][tap][Cin] fp16 -> slab images [n tile][tap][chunk][b_stride bytes]; inside a
// slab row r (output channel) holds BK channels, its 16-byte piece c sits at the K-major swizzled position the
// wgmma descriptor expects: c ^ (r & 7) for 128-byte rows, c ^ ((r >> 1) & 3) for 64-byte, c ^ ((r >> 2) & 1) for 32-byte.
__global__ void pack_weights_kernel(const __half* __restrict__ w, uint8_t* __restrict__ out, int n_tile, int n_tiles,
                                    int taps, int chunks, int BK, int Cin, uint32_t b_stride, long long pieces) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= pieces) return;
  const int c16 = BK / 8;
  const int c = (int)(i % c16);
  long long q = i / c16;
  const int r = (int)(q % n_tile); q /= n_tile;
  const int ch = (int)(q % chunks); q /= chunks;
  const int t = (int)(q % taps);
  const int nt = (int)(q / taps);
  const size_t K = (size_t)taps * Cin;
  if (ch * BK + c * 8 >= Cin) return;  // ragged last slab: stays zero
  const int4 v = *reinterpret_cast<const int4*>(w + (size_t)(nt * n_tile + r) * K + (size_t)t * Cin + ch * BK + c * 8);
  const uint32_t sw = row_swizzle_xor((uint32_t)r, (uint32_t)BK * 2);
  uint8_t* slab = out + (size_t)((nt * taps + t) * chunks + ch) * b_stride;
  *reinterpret_cast<int4*>(slab + (size_t)r * BK * 2 + ((c ^ sw) << 4)) = v;
}

// ------------------------------------------------------------------------------------------
// Host side: tiling choice + tensor maps
// ------------------------------------------------------------------------------------------
EncodeTiledFn tmap_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess ||
      qres != cudaDriverEntryPointSuccess || !p) {
    cudaGetLastError();
    return nullptr;
  }
  fn = (EncodeTiledFn)p;
  return fn;
}

int sm_count() {
  static std::mutex mu;
  static std::map<int, int> num_sms;
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> lock(mu);
  int& n = num_sms[dev];
  if (!n) cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  return n;
}

CUresult tmap_nhwc(CUtensorMap* map, CUtensorMapDataType type, void* base, int coff, int C, int W, int H, int N, int pitch,
                   const cuuint32_t* box, const cuuint32_t* estr, CUtensorMapSwizzle swz) {
  const EncodeTiledFn encode = tmap_encode_fn();
  if (!encode) return CUDA_ERROR_NOT_FOUND;
  const cuuint64_t esz = type == CU_TENSOR_MAP_DATA_TYPE_FLOAT32 ? 4 : 2;
  const cuuint64_t gdim[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  const cuuint64_t gstr[3] = {pitch * esz, pitch * esz * W, pitch * esz * W * H};
  return encode(map, type, 4, static_cast<uint8_t*>(base) + coff * esz, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

cudaError_t smem_limit(const void* kernel, size_t smem, bool max_carveout) {
  static std::mutex mu;
  static std::map<std::pair<int, const void*>, size_t> limit;
  int dev = 0;
  cudaGetDevice(&dev);
  if (max_carveout) cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  std::lock_guard<std::mutex> lock(mu);
  size_t& lim = limit[{dev, kernel}];
  if (smem <= lim) return cudaSuccess;
  const cudaError_t ce = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (ce == cudaSuccess) lim = smem;
  return ce;
}

bool tc_conv_supported(const ConvParams& p) {
  if (p.Cin % 16 || p.Cout % 16 || p.Cout > TC_MAX_COUT) return false;
  if (!((p.k == 1 && p.stride == 1) || (p.k == 3 && (p.stride == 1 || p.stride == 2)))) return false;
  if (p.in.coff % 8 || p.in.pitch % 8 || p.out.coff % 8 || p.out.pitch % 8) return false;
  if (p.res.base && (p.res.coff % 8 || p.res.pitch % 8)) return false;
  return true;
}

static int pick_n_tile(int cout) {
  if (cout <= 256) return cout;
  int best = 16;
  for (int n = 16; n <= 256; n += 16)
    if (cout % n == 0) best = n;
  return best;
}

// Operand rings of a plan: stages, resident weights, CTAs per SM and dynamic shared memory.  `extra` bytes of the budget
// hold the resident weights of a folded 1x1 (tc_fold_plan_create), placed after the rings at args.w2_off.  Returns
// false when the tile does not fit.
// Two CTAs per SM (each <= ~100 KiB smem) double the tiles in flight per SM and hide the producer -> MMA ->
// epilogue hand-off latencies of the HBM-bound high-resolution layers; they need n_tile <= 64 (the register budget of
// two 288-thread CTAs leaves room for 32 accumulator registers per thread).  Layers whose resident weights or wide N
// tiles do not fit run one CTA per SM with the full budget.
static bool tc_size_rings(TcConvPlan* plan, size_t extra, int max_occ) {
  TcArgs& a = plan->args;
  const ConvParams& p = plan->p;
  const int num_sms = sm_count();
  const size_t b_all = (size_t)a.ksteps * a.b_stride;
  const int m_tiles = plan->flat ? (p.B * p.Ho * p.Wo + 127) / 128
                                 : p.B * ((p.Wo + a.BW - 1) / a.BW) * ((p.Ho + a.BH - 1) / a.BH);
  const size_t full = 200 * 1024 > extra ? 200 * 1024 - extra : 0;  // one CTA per SM
  plan->occ = 1;
  a.stages_a = 0;
  for (int occ = 2; occ >= 1; occ--) {
    const size_t budget = occ == 2 ? (104 * 1024 > extra ? 104 * 1024 - extra : 0) : full;  // operand rings
    // layers with <= 2 tiles per CTA gain nothing from deep rings or resident weights; a small footprint
    // lets the NEXT kernel's CTAs (PDL / sibling branches) become resident while this one drains
    const bool small = m_tiles * a.n_tiles <= 2 * num_sms;
    if (occ == 2 && (a.n_tile > 64 || max_occ < 2)) continue;
    // keep the whole weight matrix in smem when it leaves room for >= 3 activation slabs: removes the
    // weight re-fetch per tile
    a.b_resident = (a.n_tiles == 1 && b_all + 3 * (size_t)a.a_stride <= budget) ? 1 : 0;
    // resident weights at one CTA/SM beat re-fetched weights at two CTAs/SM
    if (occ == 2 && !small && !a.b_resident && a.n_tiles == 1 && b_all + 3 * (size_t)a.a_stride <= full) continue;
    if (a.b_resident) {
      a.stages_a = (int)std::min<size_t>(a.mode != TC_TAP ? (a.chunks > 1 ? 8 : 6) : TC_MAX_STAGES, (budget - b_all) / a.a_stride);
      a.stages_b = 0;
    } else if (a.mode != TC_TAP) {
      // A slab serves 9 B slabs: a short A ring and as many weight slabs as fit
      a.stages_a = (int)std::min<size_t>(3, std::max<size_t>(2, (budget / 3) / a.a_stride));
      const size_t rest = budget > (size_t)a.stages_a * a.a_stride ? budget - (size_t)a.stages_a * a.a_stride : 0;
      a.stages_b = (int)std::min<size_t>(TC_MAX_STAGES, rest / a.b_stride);
    } else {
      a.stages_a = a.stages_b = (int)std::min<size_t>(8, budget / (a.a_stride + a.b_stride));
    }
    const size_t rings = (size_t)a.stages_a * a.a_stride + (a.b_resident ? b_all : (size_t)a.stages_b * a.b_stride);
    a.w2_off = (uint32_t)rings;
    plan->smem = rings + extra + 1024;
    const bool fits = a.stages_a >= 2 && (a.b_resident || a.stages_b >= ((occ == 2 && a.mode != TC_TAP) ? 3 : 2)) && rings <= budget;
    if (fits && (occ == 1 || small || a.stages_a >= 3)) { plan->occ = occ; break; }
    if (occ == 1) a.stages_a = 0;  // reported below
  }
  plan->small = m_tiles * a.n_tiles <= 2 * num_sms;
  plan->grid = num_sms * plan->occ;
  return !(a.stages_a < 2 || (!a.b_resident && a.stages_b < 2));
}

// Shared-memory limit of a conv_tc_kernel plan's instantiation (smem_limit).  false (and *err) on failure.
static bool tc_kernel_attrs(const TcConvPlan* plan, std::string* err) {
  const cudaError_t ce = smem_limit((const void*)plan->kernel, plan->smem, true);
  if (ce != cudaSuccess && err) *err = std::string("cudaFuncSetAttribute(conv_tc_kernel) failed: ") + cudaGetErrorString(ce);
  return ce == cudaSuccess;
}

TcConvPlan* tc_conv_plan_create(const ConvParams& p, std::string* err) {
  TcPlanPtr plan(new TcConvPlan());
  plan->p = p;
  TcArgs& a = plan->args;
  memset(&a, 0, sizeof(a));
  a.out = reinterpret_cast<__half*>(p.out.base);
  a.res = reinterpret_cast<const __half*>(p.res.base);
  a.bias = p.bias;
  a.out_pitch = p.out.pitch; a.out_coff = p.out.coff;
  a.res_pitch = p.res.pitch; a.res_coff = p.res.coff;
  a.ksz = p.k; a.stride = p.stride; a.pad = p.pad;
  a.Cin = p.Cin;
  // stride-2 3x3 convs over a whole-buffer view with <= 32 channels use pair rows (below)
  const bool s2p_ok = p.k == 3 && p.stride == 2 && p.in.coff == 0 && p.in.pitch == p.Cin && p.Cin <= 32 && p.in.W % 2 == 0;
  a.mode = (p.k == 3 && p.stride == 1) ? TC_HALO : (s2p_ok ? TC_S2P : TC_TAP);
  // channel slab: the widest of 64 / 32 / 16 channels (128 / 64 / 32-byte operand rows) that pads K by at most
  // 35 %; a ragged last slab
  // is zero-filled by TMA (activations, dim 0 bound = Cin) and by the weight packing.  (Wider rows mean fewer, longer
  // MMA K steps per slab.)
  auto padded = [&](int bk) { return (p.Cin + bk - 1) / bk * bk; };
  a.BK = padded(64) * 100 <= p.Cin * 135 ? 64 : (padded(32) * 100 <= p.Cin * 135 ? 32 : 16);  // <= 35 % zero K
  a.chunks = (p.Cin + a.BK - 1) / a.BK;
  a.act = p.act;
  a.n_tile = pick_n_tile(p.Cout);
  a.n_tiles = p.Cout / a.n_tile;
  a.row_bytes = a.BK * 2;
  a.layout_a = a.layout_b = row_layout(a.row_bytes);
  a.sbo_a = a.sbo_b = (8 * a.row_bytes) >> 4;

  // the input as a 4-D NHWC tensor map {C, W, H, N}: the view itself, or re-shaped below
  plan->flat = (p.k == 1 && p.stride == 1);
  int mC = p.Cin, mW = p.in.W, mH = p.in.H, mN = p.B, m_pitch = p.in.pitch, m_row_bytes = a.row_bytes;
  cuuint32_t box[4] = {(cuuint32_t)a.BK, 0, 0, 1}, estr[4] = {1, 1, 1, 1};
  if (plan->flat) {
    // all pixels of the batch form one dimension: tiles of 128 consecutive pixels
    mW = p.B * p.in.H * p.in.W; mH = mN = 1;
    a.BW = 128; a.BH = 1;
    box[1] = 128; box[2] = 1;
  } else if (a.mode == TC_HALO) {
    // 8 x 16 output pixels; one TMA box carries the 10 x 18 input halo of a channel slab
    a.BW = HALO_BW; a.BH = HALO_BH;
    a.sbo_a = ((a.BW + 2) * a.row_bytes) >> 4;
    box[1] = a.BW + 2; box[2] = a.BH + 2;
  } else if (a.mode == TC_S2P) {
    // stride-2 3x3, pair rows: two horizontally adjacent pixels (input columns 2q, 2q+1) are contiguous in a
    // whole-buffer NHWC view, so the tensor map declares them as ONE row of 2*Cin channels with the swizzle of
    // that width.  One dense box of (2BH+1) input rows x (BW+1) pairs then serves all 9 taps as row / K-slice
    // shifts (see tc_mainloop); the left / top zero padding is TMA out-of-bounds fill of pair -1 / row -1.
    // (A strided box per tap moves 9 x 128 rows of Cin*2 bytes per tile and is bound by the TMA row rate.)
    // 8 x 16 output pixels from 9 pairs x 33 input rows; consecutive output rows are two input rows = 18 pair rows apart
    a.BW = HALO_BW; a.BH = HALO_BH;
    a.sbo_a = (2 * (a.BW + 1) * 2 * a.row_bytes) >> 4;
    mC = 2 * p.Cin; mW = p.in.W / 2; m_pitch = 2 * p.in.pitch; m_row_bytes = 2 * a.row_bytes;
    a.layout_a = row_layout(m_row_bytes);
    box[0] = 2 * a.BK; box[1] = a.BW + 1; box[2] = 2 * a.BH + 1;
  } else {
    // choose the output rectangle BW x BH (<= 128 rows) with the least padding waste
    double best = -1;
    for (int bw = 1; bw <= std::min(p.Wo, 128); bw++) {
      const int bh = std::min(p.Ho, 128 / bw);
      if (bw * p.stride > 256 || bh * p.stride > 256) continue;
      const double tiles = (double)((p.Wo + bw - 1) / bw) * ((p.Ho + bh - 1) / bh);
      const double eff = (double)p.Wo * p.Ho / (tiles * 128.0);
      if (eff > best + 1e-9 || (eff > best - 1e-9 && bw > a.BW)) { best = eff; a.BW = bw; a.BH = bh; }
    }
    box[1] = a.BW * p.stride; box[2] = a.BH * p.stride;
    estr[1] = estr[2] = p.stride;
  }
  const CUresult cr = tmap_nhwc(&a.tmA, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, p.in.base, p.in.coff, mC, mW, mH, mN, m_pitch, box, estr,
                                row_swizzle(m_row_bytes));
  if (cr != CUDA_SUCCESS) {
    if (err) *err = "cuTensorMapEncodeTiled(A) failed with code " + std::to_string((int)cr);
    return nullptr;
  }
  const int a_rows = a.mode == TC_HALO ? (a.BW + 2) * (a.BH + 2)
                                       : (a.mode == TC_S2P ? 2 * (a.BW + 1) * (2 * a.BH + 1) : a.BW * a.BH);
  a.a_bytes = (uint32_t)(a_rows * a.row_bytes);
  a.b_bytes = (uint32_t)(a.n_tile * a.row_bytes);
  a.a_stride = (uint32_t)((std::max(a_rows, 128) * a.row_bytes + 1023) / 1024 * 1024);
  a.b_stride = (uint32_t)((a.n_tile * a.row_bytes + 1023) / 1024 * 1024);
  a.ksteps = p.k * p.k * a.chunks;
  {
    // Weights are constant: store every [n_tile x BK] slab in global memory exactly as it must look in shared
    // memory (swizzled rows, padded to b_stride), so the kernel fetches a slab with ONE contiguous bulk copy.
    // (As 2-D TMA boxes the slabs would cost the TMA unit one row each - 7200 rows per tile for a 3x3 160->160 layer.)
    const size_t total = (size_t)a.n_tiles * a.ksteps * a.b_stride;
    if (cudaMalloc(&plan->wpk, total) != cudaSuccess) {
      if (err) *err = "cudaMalloc(packed weights) failed";
      cudaGetLastError();
      plan->wpk = nullptr;
      return nullptr;
    }
    cudaMemset(plan->wpk, 0, total);
    const int chunks16 = a.BK / 8;  // 16-byte pieces per row
    const long long pieces = (long long)a.n_tiles * a.ksteps * a.n_tile * chunks16;
    pack_weights_kernel<<<(unsigned)((pieces + 255) / 256), 256>>>(reinterpret_cast<const __half*>(p.w), plan->wpk, a.n_tile,
                                                                    a.n_tiles, p.k * p.k, a.chunks, a.BK, p.Cin,
                                                                    a.b_stride, pieces);
    if (cudaDeviceSynchronize() != cudaSuccess) {
      if (err) *err = std::string("pack_weights_kernel failed: ") + cudaGetErrorString(cudaGetLastError());
      return nullptr;
    }
    a.wpk = plan->wpk;
  }
  if (!tc_size_rings(plan.get(), 0, tc_ctas_per_sm(a.n_tile / 16, 0))) {
    if (err) *err = "tile does not fit in shared memory";
    return nullptr;
  }
  a.epi_mode = p.dec.mode;
  a.dA = p.dec.A; a.dCtot = p.dec.Ctot; a.da0 = p.dec.a0; a.dch0 = p.dec.ch0; a.dWl = p.dec.Wl; a.dHW = p.dec.HW;
  a.dstride = p.dec.stride;
  if (a.epi_mode != EPI_STORE && !(plan->flat && a.n_tiles == 1 && (a.epi_mode != EPI_DFL_BOX || a.n_tile == 64))) {
    if (err) *err = "fused decode epilogue needs a flattened 1x1 conv with a single N tile";
    return nullptr;
  }
  dispatch_nt16(a.n_tile / 16, [&](auto nt16) { plan->kernel = conv_tc_kernel<decltype(nt16)::value>; });
  if (!tc_kernel_attrs(plan.get(), err)) return nullptr;
  return plan.release();
}

// The fold instantiations, as (this conv's n_tile, the 1x1's Cout) / 16: the pairs of the YOLOv8 / YOLOv11 detection
// models.  A pair without one stays unfolded; 256 -> 128 and 160 -> 160 are left out because their fragments and
// accumulators spill even at one CTA per SM (the 1x1 passes of 64 / 80 columns need the fragments of all 256 / 160
// input channels live through every pass).
static void (*tc_fold_kernel(int nt16, int n2_16))(TcArgs) {
#define YB_FOLD_KERNEL(N, N2) \
  if (nt16 == N && n2_16 == N2) return conv_tc_kernel<N, N2>;
  YB_FOLD_KERNEL(2, 2)    // 32 -> 32: v8n / v11n model.1 -> model.2.cv1
  YB_FOLD_KERNEL(4, 4)    // 64 -> 64: model.1 / 3 -> C2f / C3k2 cv1, the DFL box tails of c2 = 64
  YB_FOLD_KERNEL(5, 4)    // 80 -> 64: DFL box tails of c2 = 80 (v8x)
  YB_FOLD_KERNEL(5, 5)    // 80 -> 80: class tails of c3 = 80 (v8n, v11n)
  YB_FOLD_KERNEL(8, 5)    // 128 -> 80: class tails of c3 = 128 (v8s, v11s)
  YB_FOLD_KERNEL(8, 8)    // 128 -> 128: model.5 -> model.6.cv1 (v8n), model.3 -> model.4.cv1 (v8s)
#undef YB_FOLD_KERNEL
  return nullptr;
}

TcConvPlan* tc_fold_plan_create(const TcConvPlan* pa, const TcConvPlan* pb, std::string* err) {
  const TcArgs &a1 = pa->args, &a2 = pb->args;
  const ConvParams &p1 = pa->p, &p2 = pb->p;
  auto fail = [&](const std::string& m) -> TcConvPlan* { if (err) *err = m; return nullptr; };
  if (a1.n_tiles != 1) return fail("the producer splits Cout over " + std::to_string(a1.n_tiles) + " N tiles");
  if (a1.epi_mode != EPI_STORE || p1.res.base || (p1.act != ACT_SILU && p1.act != ACT_NONE))
    return fail("the producer is not a plain conv that stores its output");
  if (!pb->flat || a2.n_tiles != 1 || p2.res.base || p2.Cin != p1.Cout || p2.Cout > TC_FOLD_BIAS)
    return fail("the consumer is not a single-tile 1x1 over the producer's channels");
  const int nt16 = a1.n_tile / 16, n2_16 = p2.Cout / 16;
  // column passes of at most 80: the second accumulator stays within the register budget of the producer's tile
  const int f16 = tc_fold_pass16(n2_16);
  TcPlanPtr plan(new TcConvPlan(*pa));
  plan->wpk = nullptr;  // both slab sets belong to the two conv plans
  plan->fold16 = f16;
  TcArgs& a = plan->args;
  a.w2 = a2.wpk; a.bias2 = p2.bias;
  a.w2_bytes = (uint32_t)(a2.ksteps * a2.b_stride);
  a.b2_stride = a2.b_stride; a.sbo_b2 = a2.sbo_b; a.layout_b2 = a2.layout_b;
  a.BK2 = a2.BK; a.n2 = p2.Cout; a.act1 = a1.act;
  // the epilogue is the 1x1's
  a.out = a2.out; a.out_pitch = a2.out_pitch; a.out_coff = a2.out_coff;
  a.res = nullptr; a.res_pitch = a.res_coff = 0;
  a.act = a2.act;
  a.epi_mode = a2.epi_mode;
  a.dA = a2.dA; a.dCtot = a2.dCtot; a.da0 = a2.da0; a.dch0 = a2.dch0; a.dWl = a2.dWl; a.dHW = a2.dHW; a.dstride = a2.dstride;
  if (!tc_size_rings(plan.get(), a.w2_bytes, tc_ctas_per_sm(nt16, n2_16)))
    return fail("the producer's rings and the 1x1's " + std::to_string(a.w2_bytes / 1024) + " KiB of weights do not fit in shared memory");
  plan->kernel = tc_fold_kernel(nt16, n2_16);
  if (!plan->kernel || (a2.epi_mode == EPI_DFL_BOX && f16 != 4))
    return fail("no fold instantiation for " + std::to_string(a1.n_tile) + " -> " + std::to_string(p2.Cout) + " channels");
  if (!tc_kernel_attrs(plan.get(), err)) return nullptr;
  return plan.release();
}

std::string tc_conv_plan_describe(const TcConvPlan* plan) {
  const TcArgs& a = plan->args;
  char buf[320];
  int n = snprintf(buf, sizeof(buf), "mode %d BK %d chunks %d n_tile %d x%d stages a/b %d/%d resident %d occ %d threads %d smem %zu KiB grid %d",
                   a.mode, a.BK, a.chunks, a.n_tile, a.n_tiles, a.stages_a, a.stages_b, a.b_resident, plan->occ, TC_THREADS,
                   plan->smem / 1024, plan->grid);
  if (plan->fold16 && n > 0 && n < (int)sizeof(buf))
    snprintf(buf + n, sizeof(buf) - n, " fold 1x1 %d->%d BK %d pass %d w2 %u KiB", a.n_tile, a.n2, a.BK2, 16 * plan->fold16,
             a.w2_bytes / 1024);
  return buf;
}

void tc_conv_plan_destroy(TcConvPlan* plan) {
  if (plan && plan->wpk) cudaFree(plan->wpk);
  delete plan;
}

long long* g_tc_dbg = nullptr;  // set by yb_debug_timeline: next tensor-core conv launches write their timeline here
int g_tc_dbg_countdown = -1;

int tc_conv_launch(const TcConvPlan* plan, int B, float* pred, int* tile_ctr, cudaStream_t s) {
  TcArgs a = plan->args;
  a.pred = pred;
  a.tile_ctr = tile_ctr;
  a.dbg = nullptr;
  if (g_tc_dbg && g_tc_dbg_countdown >= 0 && g_tc_dbg_countdown-- == 0) a.dbg = g_tc_dbg;
  const ConvParams& p = plan->p;
  if (plan->flat) {  // 128-pixel tiles of the flattened batch (BW = 128, BH = 1)
    a.imgs = 1;
    a.Ho = 1;
    a.Wo = B * p.Ho * p.Wo;
  } else {
    a.imgs = B;
    a.Ho = p.Ho; a.Wo = p.Wo;
  }
  a.tg = tile_grid(a.imgs, a.Ho, a.Wo, a.BH, a.BW, a.n_tiles);
  a.m_bw = fdiv_magic(a.BW);
  int max_grid = plan->grid;
  // concurrent head branches: a latency-bound layer with ~1 tile per CTA gives up half of its CTAs (each
  // then pipelines 2-3 tiles) so that a sibling branch can occupy the other SMs at the same time
  if (plan->p.share_sms && a.tg.total <= 4 * plan->grid && a.ksteps * (a.BK >> 4) <= 40)
    max_grid = std::min(max_grid, (a.tg.total + 2) / 3);
  const int grid = tc_grid(max_grid, a.tg.total, &a.tile_batch);
  YB_CUDA_CHECK(launch_pdl(plan->kernel, dim3(grid), dim3(TC_THREADS), plan->smem, s, a));
  return 0;
}

// ------------------------------------------------------------------------------------------
// Fused Bottleneck (Block.cs:572-607 with k = (3, 3)): out = SiLU(conv_b(t) + bias_b) [+ x], t = fp16(SiLU(conv_a(x) +
// bias_a)).  t never leaves shared memory; the block input is read from HBM once and also serves as the shortcut.
//   tile      the 8 x 16 output rectangle of a halo tile (HALO_BW x HALO_BH)
//   input     one 4-D TMA box {BK1, 12, 20, 1} per channel slab at (w0 - 2, h0 - 2), zero out-of-bounds fill: box pixel
//             (h, w) sits at row 12 h + w
//   stage 1   M = box rows 0..255, four blocks of 64 (two per warpgroup), SBO = 8 rows: row 12 h + w is t pixel (h, w)
//             of the 10 x 18 halo of t when w < 10 and h < 18, i.e. 180 of the 256 MMA rows do useful work.  Tap (kh, kw)
//             is the same bytes shifted by 12 kh + kw rows (as TC_HALO); the rows that run past the box only feed the
//             discarded MMA rows.
//   t         fp16 in shared memory at the same row index (pitch 12), one slab per BK2 channels, swizzled as a TMA box of
//             that width would be; zero where its pixel lies outside the image (the zero padding of conv_b)
//   stage 2   the TC_HALO mapping over t with SBO = 12 rows, both weight sets resident
//   shortcut  the centre of the staged input box, read into registers before its ring slot is handed back
// Rounding points are those of the two unfused launches: fp32 sums, + bias, SiLU, fp16 t; the same for stage 2, then
// + residual and the fp16 store.
// ------------------------------------------------------------------------------------------
constexpr int BN_PITCH = HALO_BW + 4;               // width of the input box = row pitch of t
constexpr int BN_XROWS = BN_PITCH * (HALO_BH + 4);  // 240 rows of the input box
constexpr int BN_TROWS = BN_PITCH * (HALO_BH + 2);  // 216 rows of t (columns 10 and 11 unused)
constexpr int BN_MAX_C = 64;                        // cmid, cout: one N tile of at most 64 columns per stage
constexpr size_t BN_MAX_RINGS = 220 * 1024;         // input ring + weights + t of a one-CTA-per-SM plan (+ 1 KiB alignment)

struct BnArgs {
  CUtensorMap tmX;
  const uint8_t *w1, *w2;  // packed weight slabs of conv_a / conv_b (pack_weights_kernel, one N tile)
  const float *bias1, *bias2;
  __half* out;
  int out_pitch, out_coff;
  int shortcut;
  int H, W;
  TileGrid tg;
  int cmid, cout;
  int BK1, chunks1, BK2, chunks2;
  uint32_t layout1, layout2;          // wgmma layout types of the BK1 / BK2 rows
  uint32_t x_bytes, x_stride, slot;   // input: TMA bytes / smem bytes per channel slab; one ring slot = chunks1 slabs
  uint32_t w1_bytes, w2_bytes, b1_stride, b2_stride;
  uint32_t t_stride;                  // smem bytes per BK2-channel slab of t
  int stages;
  int* tile_ctr;
  int tile_batch;
};

struct TcBneckPlan {
  BnArgs args;
  size_t smem;
  int grid, occ;
  void (*kernel)(BnArgs) = nullptr;
};

// byte offset of (row r, byte b) in a slab of `rb`-byte swizzled rows whose base is 1 KiB aligned (pack_weights_kernel)
__device__ __forceinline__ uint32_t sw_off(uint32_t r, uint32_t b, uint32_t rb) {
  return r * rb + (((b >> 4) ^ row_swizzle_xor(r, rb)) << 4) + (b & 15);
}

// stage 1 of one warpgroup: MMA rows 128 wg .. 128 wg + 127 as two 64-row accumulators, one commit group per tile
template <int NM16, int KK>
__device__ __forceinline__ void bn_stage1(const BnArgs& a, float (&acc)[2][NM16 * 8], uint32_t xslot, uint32_t w1, int wg) {
  constexpr uint32_t RB16 = KK * 2;
  const uint32_t hi = wg_desc_hi(8 * RB16, a.layout1);
  uint32_t scale = 0;
  wg_fence();
  for (int ch = 0; ch < a.chunks1; ch++) {
    const uint32_t a_lo = wg_desc_lo(xslot + ch * a.x_stride) + (uint32_t)wg * 128 * RB16;
#pragma unroll
    for (int t = 0; t < 9; t++) {
      const uint32_t tap = tap_shift(t, BN_PITCH, RB16);
      const uint32_t b_lo = wg_desc_lo(w1 +(t * a.chunks1 + ch) * a.b1_stride);
#pragma unroll
      for (int k = 0; k < KK; k++) {
#pragma unroll
        for (int j = 0; j < 2; j++) wg_mma_n<NM16, false>(acc[j], a_lo + j * 64 * RB16 + tap + 2 * k, hi, b_lo + 2 * k, hi, RB16, scale);
        scale = 1;
      }
    }
  }
  wg_commit();
  wg_wait<0>();
  wg_fence_acc<NM16 * 8>(acc[0]);
  wg_fence_acc<NM16 * 8>(acc[1]);
}

// stage 2 of one warpgroup: output rows 64 wg.. (image rows 8 wg..) over t, SBO = one t row of 12 pixels
template <int NO16, int KK>
__device__ __forceinline__ void bn_stage2(const BnArgs& a, float* acc, uint32_t tbase, uint32_t w2, int wg) {
  constexpr uint32_t RB16 = KK * 2;
  const uint32_t a_hi = wg_desc_hi(BN_PITCH * RB16, a.layout2), b_hi = wg_desc_hi(8 * RB16, a.layout2);
  uint32_t scale = 0;
  wg_fence();
  for (int ch = 0; ch < a.chunks2; ch++) {
    const uint32_t a_lo = wg_desc_lo(tbase + ch * a.t_stride) + (uint32_t)wg * 8 * BN_PITCH * RB16;
#pragma unroll
    for (int t = 0; t < 9; t++) {
      const uint32_t tap = tap_shift(t, BN_PITCH, RB16);
      const uint32_t b_lo = wg_desc_lo(w2 +(t * a.chunks2 + ch) * a.b2_stride);
#pragma unroll
      for (int k = 0; k < KK; k++) {
        wg_mma_n<NO16, false>(acc, a_lo + tap + 2 * k, a_hi, b_lo + 2 * k, b_hi, RB16, scale);
        scale = 1;
      }
    }
  }
  wg_commit();
  wg_wait<0>();
  wg_fence_acc<NO16 * 8>(acc);
}

// CTAs per SM the register bound of each instantiation allows without spills (ptxas -v): the per-tile chain of loads,
// two MMA stages and two epilogues is latency-bound at small channel counts, so concurrent CTAs are what fills the SM
__host__ __device__ constexpr int bn_ctas_per_sm(int nm16, int no16) { return nm16 == 1 && no16 <= 2 ? 3 : (nm16 <= 2 && no16 <= 2 ? 2 : 1); }

__device__ __forceinline__ uint32_t ld_shared_u32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void st_shared_u32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 1, %0;" ::"n"(TC_CONSUMERS) : "memory"); }

template <int NM16, int NO16>
__global__ void __launch_bounds__(TC_THREADS, bn_ctas_per_sm(NM16, NO16)) bneck_tc_kernel(const __grid_constant__ BnArgs a) {
  extern __shared__ __align__(1024) uint8_t bn_smem[];
  __shared__ __align__(8) uint64_t bars[2 * TC_MAX_STAGES + 1];
  __shared__ int s_tile[TQ];
  __shared__ volatile int s_head;
  __shared__ __align__(16) float s_bias1[BN_MAX_C], s_bias2[BN_MAX_C];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < a.cmid; i += blockDim.x) s_bias1[i] = a.bias1[i];  // constant data
  for (int i = threadIdx.x; i < a.cout; i += blockDim.x) s_bias2[i] = a.bias2[i];
  const uint32_t sX = (smem_u32(bn_smem) + 1023u) & ~1023u;  // input ring, then W1, W2, t
  const uint32_t sW1 = sX + a.stages * a.slot, sW2 = sW1 + a.w1_bytes, sT = sW2 + a.w2_bytes;
  const uint32_t full = smem_u32(&bars[0]), empty = smem_u32(&bars[TC_MAX_STAGES]), wfull = smem_u32(&bars[2 * TC_MAX_STAGES]);
  // t starts zeroed: when cmid is not a multiple of BK2 (48 channels in 64-channel slabs), channels cmid.. of every row
  // are K padding that stage 2 multiplies with zero weights and the epilogue never writes - stale bytes there could be
  // Inf / NaN patterns
  for (uint32_t i = threadIdx.x; i < a.chunks2 * a.t_stride / 16; i += blockDim.x) st_shared_v4(sT + 16 * i, make_int4(0, 0, 0, 0));
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy zeros -> visible to the MMA

  pdl_trigger();
  if (warp == TC_CONSUMER_WARPS && lane == 0) {
    s_head = 0;
    for (int s = 0; s < a.stages; s++) {
      mbar_init(full + 8 * s, 1);
      mbar_init(empty + 8 * s, TC_CONSUMER_WARPS);
    }
    mbar_init(wfull, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  if (warp == TC_CONSUMER_WARPS && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&a.tmX) : "memory");
    // weights do not depend on the previous kernel: fetch them before the grid dependency resolves
    mbar_arrive_expect_tx(wfull, a.w1_bytes + a.w2_bytes);
    bulk_load_1d(sW1, a.w1, a.w1_bytes, wfull);
    bulk_load_1d(sW2, a.w2, a.w2_bytes, wfull);
  }
  pdl_wait();

  if (warp == TC_CONSUMER_WARPS) {
    // ===================== TMA producer: one ring slot (all input channel slabs) per tile =====================
    if (lane == 0) {
      int s = 0, li = 0;
      uint32_t ph = 0;
      TileDraw td(a.tile_ctr, a.tile_batch, a.tg.total);
      for (; td.tile < a.tg.total; li++) {
        tq_publish(s_tile, &s_head, li, td.tile);
        const TileCoord tc = tile_coord(a.tg, td.tile);
        mbar_wait(empty + 8 * s, ph ^ 1);
        mbar_arrive_expect_tx(full + 8 * s, a.chunks1 * a.x_bytes);
        for (int ch = 0; ch < a.chunks1; ch++)
          tma_load_4d(sX + s * a.slot + ch * a.x_stride, &a.tmX, full + 8 * s, ch * a.BK1, tc.tw * HALO_BW - 2, tc.th * HALO_BH - 2,
                      tc.img);
        ring_next(s, ph, a.stages);
        td.advance();
      }
      tq_publish(s_tile, &s_head, li, -1);  // end mark
    }
    return;
  }
  // ===================== consumers =====================
  const int wg = warp >> 2, g = lane >> 2, t4 = lane & 3;
  const uint32_t rb1 = a.BK1 * 2, rb2 = a.BK2 * 2;
  int s = 0;
  uint32_t ph = 0;
  mbar_wait(wfull, 0);
  for (int li = 0;; li++) {
    const int tile = tq_get(s_tile, &s_head, li);
    if (tile < 0) break;
    const int img = fdiv(tile, a.tg.m_tpi), r = tile - img * a.tg.tpi;
    const int th = fdiv(r, a.tg.m_tw), tw = r - th * a.tg.tiles_w;
    const int h0 = th * HALO_BH, w0 = tw * HALO_BW;
    const uint32_t xslot = sX + s * a.slot;
    mbar_wait(full + 8 * s, ph);
    float acc1[2][NM16 * 8];
    switch (a.BK1) {
      case 64: bn_stage1<NM16, 4>(a, acc1, xslot, sW1, wg); break;
      case 32: bn_stage1<NM16, 2>(a, acc1, xslot, sW1, wg); break;
      default: bn_stage1<NM16, 1>(a, acc1, xslot, sW1, wg); break;
    }
    // shortcut: this thread's stage-2 rows are box pixels (hl + 2, wl + 2); read before the slot is handed back
    uint32_t res[2][NO16 * 2];
    if (a.shortcut) {
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int row = wg * 64 + (warp & 3) * 16 + g + 8 * h;
        const uint32_t xr = (uint32_t)(((row >> 3) + 2) * BN_PITCH + (row & 7) + 2);
#pragma unroll
        for (int J = 0; J < NO16 * 2; J++) {
          const int c = 8 * J + 2 * t4;
          res[h][J] = ld_shared_u32(xslot + (c / a.BK1) * a.x_stride + sw_off(xr, (c % a.BK1) * 2, rb1));
        }
      }
      // these generic-proxy reads must be performed before the producer's TMA (async proxy) refills the slot
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(empty + 8 * s);
    ring_next(s, ph, a.stages);
    // t of the previous tile is free: every warpgroup retired its stage-2 MMAs before reaching this point
    consumers_sync();
#pragma unroll
    for (int j = 0; j < 2; j++)
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int row = (2 * wg + j) * 64 + (warp & 3) * 16 + g + 8 * h;
        const int hh = row / BN_PITCH, ww = row - hh * BN_PITCH;
        if (row >= BN_TROWS || ww >= HALO_BW + 2) continue;
        const int y = h0 - 1 + hh, x = w0 - 1 + ww;
        const bool inside = y >= 0 && y < a.H && x >= 0 && x < a.W;
#pragma unroll
        for (int J = 0; J < NM16 * 2; J++) {
          const int c = 8 * J + 2 * t4;
          float2 f = make_float2(0.f, 0.f);
          if (inside) {
            const float2 b = *reinterpret_cast<const float2*>(s_bias1 + c);
            f.x = silu_tanh(acc1[j][4 * J + 2 * h] + b.x);
            f.y = silu_tanh(acc1[j][4 * J + 2 * h + 1] + b.y);
          }
          const __half2 v = __floats2half2_rn(f.x, f.y);
          st_shared_u32(sT + (c / a.BK2) * a.t_stride + sw_off((uint32_t)row, (c % a.BK2) * 2, rb2),
                        *reinterpret_cast<const uint32_t*>(&v));
        }
      }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy t writes -> visible to the MMA
    consumers_sync();
    float acc2[NO16 * 8];
    switch (a.BK2) {
      case 64: bn_stage2<NO16, 4>(a, acc2, sT, sW2, wg); break;
      case 32: bn_stage2<NO16, 2>(a, acc2, sT, sW2, wg); break;
      default: bn_stage2<NO16, 1>(a, acc2, sT, sW2, wg); break;
    }
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int row = wg * 64 + (warp & 3) * 16 + g + 8 * h;
      const int y = h0 + (row >> 3), x = w0 + (row & 7);
      if (y >= a.H || x >= a.W) continue;
      __half* orow = a.out + ((size_t)(img * a.H + y) * a.W + x) * a.out_pitch + a.out_coff;
#pragma unroll
      for (int J = 0; J < NO16 * 2; J++) {
        const int c = 8 * J + 2 * t4;
        float2 f = bias_act(acc2 + 4 * J + 2 * h, s_bias2 + c, true);
        if (a.shortcut) {
          const float2 xv = __half22float2(*reinterpret_cast<const __half2*>(&res[h][J]));
          f.x += xv.x; f.y += xv.y;
        }
        *reinterpret_cast<__half2*>(orow + c) = __floats2half2_rn(f.x, f.y);
      }
    }
  }
}

TcBneckPlan* tc_bneck_plan_create(const TcConvPlan* pa, const TcConvPlan* pb, std::string* err) {
  const ConvParams &p1 = pa->p, &p2 = pb->p;
  const TcArgs &a1 = pa->args, &a2 = pb->args;
  auto fail = [&](const char* m) -> TcBneckPlan* { if (err) *err = m; return nullptr; };
  if (a1.mode != TC_HALO || a2.mode != TC_HALO || a1.n_tiles != 1 || a2.n_tiles != 1 || p1.Cout != p2.Cin ||
      p1.Cout > BN_MAX_C || p2.Cout > BN_MAX_C || p1.act != ACT_SILU || p2.act != ACT_SILU || p1.res.base ||
      a1.epi_mode != EPI_STORE || a2.epi_mode != EPI_STORE)
    return fail("not a fusable 3x3 / 3x3 pair");
  const bool shortcut = p2.res.base != nullptr;
  if (shortcut && (p2.res.base != p1.in.base || p2.res.coff != p1.in.coff || p2.res.pitch != p1.in.pitch || p1.Cin != p2.Cout))
    return fail("shortcut is not the block input");
  std::unique_ptr<TcBneckPlan> plan(new TcBneckPlan());
  BnArgs& a = plan->args;
  memset(&a, 0, sizeof(a));
  const cuuint32_t box[4] = {(cuuint32_t)a1.BK, (cuuint32_t)BN_PITCH, (cuuint32_t)(HALO_BH + 4), 1}, estr[4] = {1, 1, 1, 1};
  if (tmap_nhwc(&a.tmX, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, p1.in.base, p1.in.coff, p1.Cin, p1.in.W, p1.in.H, p1.B, p1.in.pitch, box,
                estr, row_swizzle(a1.BK * 2)) != CUDA_SUCCESS)
    return fail("cuTensorMapEncodeTiled(bottleneck input) failed");
  a.w1 = a1.wpk; a.w2 = a2.wpk;
  a.bias1 = p1.bias; a.bias2 = p2.bias;
  a.out = reinterpret_cast<__half*>(p2.out.base);
  a.out_pitch = p2.out.pitch; a.out_coff = p2.out.coff;
  a.shortcut = shortcut;
  a.H = p2.Ho; a.W = p2.Wo;
  a.cmid = p1.Cout; a.cout = p2.Cout;
  a.BK1 = a1.BK; a.chunks1 = a1.chunks; a.layout1 = a1.layout_a;
  a.BK2 = a2.BK; a.chunks2 = a2.chunks; a.layout2 = a2.layout_a;
  auto kib = [](size_t b) { return (uint32_t)((b + 1023) / 1024 * 1024); };
  a.x_bytes = (uint32_t)(BN_XROWS * a.BK1 * 2);
  a.x_stride = kib(a.x_bytes);
  a.slot = a.chunks1 * a.x_stride;
  a.b1_stride = a1.b_stride; a.b2_stride = a2.b_stride;
  a.w1_bytes = (uint32_t)(a1.ksteps * a1.b_stride);
  a.w2_bytes = (uint32_t)(a2.ksteps * a2.b_stride);
  a.t_stride = kib((size_t)BN_TROWS * a.BK2 * 2);
  const size_t fixed = (size_t)a.w1_bytes + a.w2_bytes + (size_t)a.chunks2 * a.t_stride;
  // as many CTAs per SM as the kernel's register bound allows and their rings fit; otherwise one CTA with as deep an
  // input ring as the remaining shared memory holds (one slot at c = 64: the input slot is handed back right after
  // stage 1, so the next tile's load still overlaps stage 2)
  const int nm16 = a.cmid / 16, no16 = a.cout / 16;
  plan->occ = 0;
  for (int occ = bn_ctas_per_sm(nm16, no16); occ >= 1 && !plan->occ; occ--) {
    const size_t budget = occ == 3 ? 72 * 1024 : (occ == 2 ? 104 * 1024 : BN_MAX_RINGS);
    if (fixed >= budget) continue;
    a.stages = (int)std::min<size_t>(4, (budget - fixed) / a.slot);
    if (a.stages >= occ) plan->occ = occ;
  }
  if (!plan->occ) return fail("bottleneck tile does not fit in shared memory");
  // At one CTA per SM both stages and their epilogues run back to back with nothing to overlap them, and without a
  // shortcut the launch saves only the round trip of t: the two unfused launches measure as fast (v8n c = 64 on H100)
  // and the forward faster, so such a pair stays unfused.
  if (plan->occ == 1 && !shortcut) return fail("one CTA per SM and no shortcut: the unfused pair is as fast");
  plan->smem = (size_t)a.stages * a.slot + fixed + 1024;
  dispatch_nt16(nm16, [&](auto m) {
    dispatch_nt16(no16, [&](auto o) {
      constexpr int M = decltype(m)::value, O = decltype(o)::value;
      if constexpr (M <= BN_MAX_C / 16 && O <= BN_MAX_C / 16) plan->kernel = bneck_tc_kernel<M, O>;
    });
  });
  if (smem_limit((const void*)plan->kernel, plan->smem, true) != cudaSuccess) return fail("cudaFuncSetAttribute(bneck_tc_kernel) failed");
  plan->grid = sm_count() * plan->occ;
  return plan.release();
}

std::string tc_bneck_plan_describe(const TcBneckPlan* plan) {
  const BnArgs& a = plan->args;
  char buf[256];
  snprintf(buf, sizeof(buf), "fused bottleneck %d->%d BK %d/%d chunks %d/%d shortcut %d stages %d occ %d smem %zu KiB grid %d",
           a.cmid, a.cout, a.BK1, a.BK2, a.chunks1, a.chunks2, a.shortcut, a.stages, plan->occ, plan->smem / 1024, plan->grid);
  return buf;
}

void tc_bneck_plan_destroy(TcBneckPlan* plan) { delete plan; }  // the weight slabs belong to the two conv plans

int tc_bneck_launch(const TcBneckPlan* plan, int B, int* tile_ctr, cudaStream_t s) {
  BnArgs a = plan->args;
  a.tg = tile_grid(B, a.H, a.W, HALO_BH, HALO_BW, 1);
  a.tile_ctr = tile_ctr;
  const int grid = tc_grid(plan->grid, a.tg.total, &a.tile_batch);
  YB_CUDA_CHECK(launch_pdl(plan->kernel, dim3(grid), dim3(TC_THREADS), plan->smem, s, a));
  return 0;
}

// ------------------------------------------------------------------------------------------
// Stem: model.0 = Conv(3, C, k3, s2) straight from the NCHW network input (u8 / f16 / f32) on the tensor
// cores.  K ordering is chosen so that im2col needs no element shuffling: for output pixel (ho, wo) and each
// of the 9 (kh, c) input rows, the FOUR contiguous input columns 2wo-2 .. 2wo+1 form one 8-byte K group
//     k = (kh*3 + c)*4 + slot,   slot 0 -> column 2wo-2 (weight 0), slots 1..3 -> kw = 0..2
// so a thread builds its A row from 9 aligned 8-byte loads (K = 36, padded to 48 = 3 MMAs) instead of 27
// scalar loads + repacking.
//   A tile   128 rows x 128 B, SWIZZLE_128B layout written by hand (16-byte piece p of row r at p ^ (r & 7))
//   weights  [Cout][64] fp16 resident in smem, same layout
//   MMA      the same warpgroup: wgmma m64nNk16 for rows 0-63 and 64-127, K = 3 x 16, N = 64 output channels
//            per pass (fewer in the last pass), fp32 accumulators in registers
//   epilogue same 128 threads: +bias -> SiLU -> fp16 NHWC stores
// Four CTAs per SM overlap each other's load / MMA / store latencies; the layer is HBM-bound
// (reads the image once, writes Cout x H/2 x W/2 fp16).
// ------------------------------------------------------------------------------------------
constexpr int ST_TW = 16, ST_TH = 8;
constexpr int ST_THREADS = 128;  // one warpgroup: im2col, MMA and epilogue

struct StemArgs {
  const void* in;
  const __half* w16;   // [Cout][64] fp16, k = (kh*3 + c)*4 + kw + 1, other k zero
  const float* bias;
  __half* out;
  int out_pitch, out_coff;
  int B, H, W, Ho, Wo, Cout;
  // Detector.ImagePredict pads the image right / bottom to a multiple of 32 with the value 114 before the /255
  // (Models/Detector.cs:35-41): the caller's tensor is (B, 3, src_H, src_W) with src <= H, W and the padding is
  // produced here instead of by a separate pad kernel.  pad_h2 = the padded pixel as two fp16 (already scaled).
  int src_H, src_W;
  uint32_t pad_h2;
  TileGrid tg;
};

// four input columns col .. col+3 (col even, may be -2) of one row as 4 halves; `lo_ok` = col >= 0
template <int DT>
__device__ __forceinline__ uint2 stem_load4(const void* in, size_t rowbase, int col, bool lo_ok) {
  uint2 r = make_uint2(0u, 0u);
  if (DT == YB_F16) {
    const uint32_t* p = reinterpret_cast<const uint32_t*>(reinterpret_cast<const __half*>(in) + rowbase + col);
    if (lo_ok) r.x = __ldg(p);
    r.y = __ldg(p + 1);
  } else if (DT == YB_U8) {
    // two bytes -> half2 without integer->float conversions: 0x6400 | b is the fp16 number 1024 + b, and
    // fma(1024 + b, k, -1024 k) = b * k rounded once (k = fp16(1/255); Detector.cs:41 divides by 255)
    const uint16_t* p = reinterpret_cast<const uint16_t*>(reinterpret_cast<const uint8_t*>(in) + rowbase + col);
    const __half2 k2 = __float2half2_rn(1.0f / 255.0f);
    const __half2 c2 = __hmul2(k2, __float2half2_rn(-1024.0f));
    auto cvt = [&](uint32_t v) {
      const uint32_t x = __byte_perm(v, 0x64006400u, 0x7150);
      const __half2 h = __hfma2(*reinterpret_cast<const __half2*>(&x), k2, c2);
      return *reinterpret_cast<const uint32_t*>(&h);
    };
    if (lo_ok) r.x = cvt(__ldg(p));
    r.y = cvt(__ldg(p + 1));
  } else {
    const float2* p = reinterpret_cast<const float2*>(reinterpret_cast<const float*>(in) + rowbase + col);
    if (lo_ok) { const float2 v = __ldg(p); r.x = pack_h2(v.x, v.y); }
    const float2 v = __ldg(p + 1);
    r.y = pack_h2(v.x, v.y);
  }
  return r;
}

// one input element as fp16 bits (same arithmetic as stem_load4)
template <int DT>
__device__ __forceinline__ uint32_t stem_load1(const void* in, size_t i) {
  if (DT == YB_F16) return (uint32_t)__ldg(reinterpret_cast<const unsigned short*>(in) + i);
  if (DT == YB_U8) {
    const __half k = __float2half_rn(1.0f / 255.0f);
    const uint32_t x = 0x6400u | (uint32_t)__ldg(reinterpret_cast<const uint8_t*>(in) + i);
    const unsigned short xs = (unsigned short)x;
    const __half h = __hfma(*reinterpret_cast<const __half*>(&xs), k, __hmul(k, __float2half_rn(-1024.0f)));
    return (uint32_t)*reinterpret_cast<const unsigned short*>(&h);
  }
  const __half h = __float2half_rn(__ldg(reinterpret_cast<const float*>(in) + i));
  return (uint32_t)*reinterpret_cast<const unsigned short*>(&h);
}

// four columns col .. col+3 of a SOURCE row that may end before them (ragged width / odd row alignment): columns
// < 0 are the conv's zero padding, columns >= src_W the 114-padding of the image
template <int DT>
__device__ __forceinline__ uint2 stem_load4_ragged(const void* in, size_t rowbase, int col, int src_W, uint32_t pad1) {
  uint32_t e[4];
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int c = col + j;
    e[j] = c < 0 ? 0u : (c >= src_W ? pad1 : stem_load1<DT>(in, rowbase + c));
  }
  return make_uint2(e[0] | (e[1] << 16), e[2] | (e[3] << 16));
}

// One pass of W (64 / 48 / 32 / 16) output channels c0.. of the current tile: 2 x 3 wgmma, then the epilogue of those
// channels.  Row r of the tile is output pixel (tx, ty) = (r % 16, r / 16).
template <int W>
__device__ __forceinline__ void stem_pass(const StemArgs& a, uint32_t smA, uint32_t smB, const float* s_bias, int c0, int n,
                                          int th, int tw) {
  float acc[2][W / 2];
  const uint32_t hi = wg_desc_hi(64, 1);  // SBO = 8 rows x 128 B, SWIZZLE_128B
  wg_fence();
#pragma unroll
  for (int h = 0; h < 2; h++)
#pragma unroll
    for (int k = 0; k < 3; k++)
      wg_mma_n<W / 16, false>(acc[h], wg_desc_lo(smA + h * 64 * 128) + 2 * k, hi, wg_desc_lo(smB + c0 * 128) + 2 * k, hi, 8,
                              k > 0 ? 1u : 0u);
  wg_commit();
  wg_wait<0>();
  wg_fence_acc<W / 2>(acc[0]);
  wg_fence_acc<W / 2>(acc[1]);
#pragma unroll
  for (int h = 0; h < 2; h++)
#pragma unroll
    for (int e = 0; e < 2; e++) {
      const int row = acc_row(h, e);
      const int ho = th * ST_TH + (row >> 4), wo = tw * ST_TW + (row & 15);
      if (ho >= a.Ho || wo >= a.Wo) continue;
      __half* o = a.out + ((size_t)(n * a.Ho + ho) * a.Wo + wo) * a.out_pitch + a.out_coff + c0;
#pragma unroll
      for (int J = 0; J < W / 8; J++) {
        const int c = 8 * J + 2 * (threadIdx.x & 3);
        const float2 f = bias_act(acc[h] + 4 * J + 2 * e, s_bias + c0 + c, true);
        *reinterpret_cast<__half2*>(o + c) = __floats2half2_rn(f.x, f.y);
      }
    }
}

template <int DT>
__global__ void __launch_bounds__(ST_THREADS, 4) stem_tc_kernel(const __grid_constant__ StemArgs a) {
  extern __shared__ __align__(1024) uint8_t st_smem[];
  __shared__ __align__(16) float s_bias[256];
  const int tid = threadIdx.x;
  const uint32_t base = (smem_u32(st_smem) + 1023u) & ~1023u;
  const uint32_t smA = base;              // 128 rows x 128 B
  const uint32_t smB = base + 16 * 1024;  // Cout rows x 128 B
  pdl_trigger();
  // weights -> smem with the SWIZZLE_128B pattern; the K padding of the A rows is zeroed once
  for (int i = tid; i < a.Cout * 8; i += ST_THREADS) {
    const int n = i >> 3, pc = i & 7;
    const int4 v = *reinterpret_cast<const int4*>(a.w16 + n * 64 + pc * 8);
    st_shared_v4(smB + n * 128 + ((pc ^ (n & 7)) << 4), v);
  }
  for (int i = tid; i < 128 * 8; i += ST_THREADS) st_shared_v4(smA + i * 16, make_int4(0, 0, 0, 0));
  for (int i = tid; i < a.Cout; i += ST_THREADS) s_bias[i] = a.bias[i];
  pdl_wait();

  const int tx = tid & (ST_TW - 1), ty = tid / ST_TW;  // output pixel of this thread's A row
  const size_t plane = (size_t)a.src_H * a.src_W;
  const bool ragged = a.src_W != a.W || a.src_H != a.H;  // padded source: rows may be misaligned and end early
  const uint32_t pad1 = a.pad_h2 & 0xffffu;
  auto gather = [&](int tile, uint2 (&v)[9]) {
    const TileCoord tc = tile_coord(a.tg, tile);
    const int n = tc.img, ho = tc.th * ST_TH + ty, wo = tc.tw * ST_TW + tx;
    const bool pix_ok = ho < a.Ho && wo < a.Wo;
    const int col = 2 * wo - 2;
#pragma unroll
    for (int kh = 0; kh < 3; kh++) {
      const int hi_ = ho * 2 + kh - 1;
      const bool row_ok = pix_ok && hi_ >= 0 && hi_ < a.H;
      const bool in_src = hi_ < a.src_H;
      const size_t rowbase = (size_t)n * 3 * plane + (size_t)((row_ok && in_src) ? hi_ : 0) * a.src_W;
#pragma unroll
      for (int c = 0; c < 3; c++) {
        uint2 g = make_uint2(0u, 0u);
        if (row_ok) {
          if (!ragged) g = stem_load4<DT>(a.in, rowbase + c * plane, col, wo > 0);
          else if (in_src) g = stem_load4_ragged<DT>(a.in, rowbase + c * plane, col, a.src_W, pad1);
          else g = make_uint2(wo > 0 ? a.pad_h2 : 0u, a.pad_h2);  // a row of the bottom padding
        }
        v[kh * 3 + c] = g;
      }
    }
  };
  uint2 v[9];
  if (blockIdx.x < a.tg.total) gather(blockIdx.x, v);
  const uint32_t a_row = smA + tid * 128;
  const uint32_t sw = (uint32_t)(tid & 7);
  for (int tile = blockIdx.x; tile < a.tg.total; tile += gridDim.x) {
    const TileCoord tc = tile_coord(a.tg, tile);
    __syncthreads();  // the previous tile's MMAs have retired in every warp before its A rows are overwritten
#pragma unroll
    for (int pc = 0; pc < 4; pc++)
      st_shared_v4(a_row + ((pc ^ sw) << 4), make_int4((int)v[2 * pc].x, (int)v[2 * pc].y, (int)v[2 * pc + 1].x, (int)v[2 * pc + 1].y));
    st_shared_v4(a_row + ((4u ^ sw) << 4), make_int4((int)v[8].x, (int)v[8].y, 0, 0));
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> visible to the MMA
    __syncthreads();
    if (tile + (int)gridDim.x < a.tg.total) gather(tile + gridDim.x, v);  // next tile's loads fly during the MMA
    for (int c0 = 0; c0 < a.Cout; c0 += 64) {
      switch (min(64, a.Cout - c0)) {
        case 64: stem_pass<64>(a, smA, smB, s_bias, c0, tc.img, tc.th, tc.tw); break;
        case 48: stem_pass<48>(a, smA, smB, s_bias, c0, tc.img, tc.th, tc.tw); break;
        case 32: stem_pass<32>(a, smA, smB, s_bias, c0, tc.img, tc.th, tc.tw); break;
        default: stem_pass<16>(a, smA, smB, s_bias, c0, tc.img, tc.th, tc.tw); break;
      }
    }
  }
}

int launch_stem_f16(const void* in, int in_dtype, int B, int H, int W, const __half* w16, const float* bias,
                    const View& out, cudaStream_t s, int src_H, int src_W) {
  if (out.C % 16 || out.C > 256 || out.coff % 8 || out.pitch % 8 || (W & 1) || (H & 1)) {
    set_error("stem: output channels must be a multiple of 16 and <= 256, input height/width even");
    return YB_ERR_SHAPE;
  }
  StemArgs a;
  memset(&a, 0, sizeof(a));
  a.in = in; a.w16 = w16; a.bias = bias;
  a.out = reinterpret_cast<__half*>(out.base);
  a.out_pitch = out.pitch; a.out_coff = out.coff;
  a.B = B; a.H = H; a.W = W; a.Ho = H / 2; a.Wo = W / 2; a.Cout = out.C;
  a.src_H = src_H > 0 ? src_H : H; a.src_W = src_W > 0 ? src_W : W;
  if (a.src_H > H || a.src_W > W) { set_error("stem: source image larger than the planned input"); return YB_ERR_SHAPE; }
  {
    // the padded pixel: u8 input -> half(114 * half(1/255)) exactly as a loaded 114 would come out; float inputs are
    // already scaled by the caller (pad(x, 114) / 255, Detector.cs:41) -> half(114 / 255)
    const __half k = __float2half_rn(1.0f / 255.0f);
    const __half pv = in_dtype == YB_U8 ? __float2half_rn(114.0f * __half2float(k)) : __float2half_rn(114.0f / 255.0f);
    const unsigned short bits = *reinterpret_cast<const unsigned short*>(&pv);
    a.pad_h2 = (uint32_t)bits | ((uint32_t)bits << 16);
  }
  a.tg = tile_grid(B, a.Ho, a.Wo, ST_TH, ST_TW, 1);
  void (*kernel)(StemArgs) = in_dtype == YB_U8 ? stem_tc_kernel<YB_U8> : (in_dtype == YB_F16 ? stem_tc_kernel<YB_F16> : stem_tc_kernel<YB_F32>);
  const size_t smem = 1024 + 16 * 1024 + (size_t)a.Cout * 128;
  YB_CUDA_CHECK(smem_limit((const void*)kernel, smem, false));
  const int grid = std::min(a.tg.total, sm_count() * 4);
  kernel<<<grid, ST_THREADS, smem, s>>>(a);
  YB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace yb
