// Halo-resident 3x3 convolution / sub-pixel ConvTranspose on Hopper wgmma (sm_90a) — the fast path for the FLOP-heavy
// stride-1 layers of the U-Net (reference ops: avatars/wav2lip/models/conv.py:5-19 Conv2d+BN+residual+ReLU and
// :33-44 ConvTranspose2d+BN+ReLU; the same kernel serves the MuseTalk VAE/UNet 3x3 convs).
//
// Idea: the nine im2col operands of a 3x3 conv are nine SHIFTED VIEWS of one input halo tile.  A CTA therefore TMA-loads
// ONE (16*NSUB+2) x 10 pixel x 64 channel halo per K chunk into shared memory (128-byte rows, SWIZZLE_128B) and addresses
// all nine views purely through the wgmma shared-memory descriptor: start address = halo + (dy*10+dx) rows, 8-row
// groups 10 rows (1280 B) apart.  The 128B swizzle is a function of the absolute smem address, so unaligned starts and
// an SBO that is not a multiple of 1024 B read exactly the rows TMA wrote.  Compared with one tile load per tap this cuts
// L2->SM operand traffic for A by 6.4x; weights are streamed 3 taps at a time and amortised over NSUB stacked 128-pixel
// sub-tiles (M = 128 * NSUB per CTA).
//
// Roles (384 threads): warps 0-7 = two consumer warpgroups, warpgroup 2 = TMA producer (one elected thread issues every
// load).  The producer warpgroup gives its registers to the consumers (setmaxnreg 40 / 232), so the accumulators and the
// epilogue of the widest tiles fit without spills.  Consumer warpgroup g owns pixel rows [8g, 8g+8) of every 16-row sub-tile
// (64 MMA rows), issues its own wgmma into register accumulators and runs the epilogue (+bias (+residual) -> ReLU -> fp16
// NHWC channel slice) straight from the accumulator fragments: the four lanes of a row swap their channel pairs so that each
// lane stores (and reads the residual of) 8 consecutive channels with one 16-byte access.  A conv whose residual is its own
// input (HaloParams::res_halo) takes it from the halo instead: the consumers ldmatrix the centre view of the chunks holding
// the tile's channels while they hold those stages, and add it in accumulator order.  Persistent CTAs: the producer runs
// ahead across tiles, so the loads of tile i+1 overlap the epilogue of tile i.
#include <cuda.h>

#include <utility>

#include "conv_halo.h"
#include "conv_tma.h"
#include "ltb_internal.h"
#include "ptx_sm90.cuh"

#ifdef LTB_HALO_DIAG
#include <cstdlib>
#define LTB_DIAG(bit) (p.dbg & (bit))
#else
#define LTB_DIAG(bit) 0
#endif

namespace ltb {

constexpr int kHaloP = 10;  // halo row pitch in pixels (8 + 2)
constexpr int kHaloThreads = 384;
constexpr int kProducerRegs = 40, kConsumerRegs = 232;   // 128 x 40 + 256 x 232 <= 64 K registers per SM
constexpr int kSms = 132;   // H100 SXM: tile-count heuristics; launches read the device's own SM count

// TAPS = 9: 3x3 conv / sub-pixel ConvT over a (16*NSUB+2) x 10 pixel halo.
// TAPS = 1: plain GEMM (1x1 conv / nn.Linear): the "halo" is the 128*NSUB-row tile itself (pitch 8 -> SBO 1024 B).
// RC > 0: "weights resident" variant for layers whose whole tap-major weight set (RC K-chunks x 9 taps x BN rows) fits
// next to the halo ring — the CTA loads it once instead of once per tile.  Requires Cout == BN.
template <int BN, int NSUB, int NACC, int TAPS, int RC = 0>
struct HaloCfg {
  static constexpr bool HALO = (TAPS != 1);                                 // 9: 3x3 conv / ConvT, 16: nearest-2x upsample + 3x3 conv
  static constexpr bool S2 = (TAPS == 10);                                  // 10: 3x3 stride-2 pad-1 conv over four parity planes
  static constexpr int P = S2 ? 9 : (HALO ? kHaloP : 8);                    // halo row pitch (pixels)
  static constexpr int HR = S2 ? 16 * NSUB + 1 : (HALO ? 16 * NSUB + 2 : 16 * NSUB);   // halo rows
  static constexpr int TG = (TAPS == 9 || TAPS == 10) ? 3 : (TAPS == 16 ? 4 : 1);      // B stages per K chunk / weight slices per B stage
  // stride 2: input pixel (2y+dy-1, 2x+dx-1) lies in parity plane (row even/odd, col even/odd); each plane is TMA-loaded with
  // traversal stride 2 into its own (HR x P) sub-tile, the nine taps are views into the four planes
  static constexpr int PLANE_BYTES = (HR * P * 128 + 1023) & ~1023;
  static constexpr int A_BYTES_RAW = (S2 ? 4 : 1) * HR * P * 128;           // TMA transaction bytes per A stage
  static constexpr int A_BYTES = S2 ? 4 * PLANE_BYTES : ((A_BYTES_RAW + 1023) & ~1023);
  static constexpr int B_BYTES = TG * BN * 128;                             // TG taps x BN rows x 64 k
  // stage counts: fill the 227 KB of shared memory
  static constexpr int BUDGET = 223 * 1024;   // 227 KB per CTA minus ~3.5 KB of static shared memory (barriers, head weights, GN table)
  static constexpr int A_STAGES_STREAM = S2 ? 2 : ((BN <= 32) ? 4 : (BN <= 64 ? 3 : (NSUB == 1 ? 3 : 2)));
  static constexpr int A_STAGES_RES = ((BUDGET - RC * TG * B_BYTES) / A_BYTES) > 4 ? 4 : ((BUDGET - RC * TG * B_BYTES) / A_BYTES);
  static constexpr int A_STAGES = RC ? A_STAGES_RES : A_STAGES_STREAM;
  // <128,2,1> reads its residual from global memory (see halo_res_smem_ok); its ring leaves room for one 128-pixel sub-tile of
  // it, so the consumers prefetch the residual while the tile's MMAs run: sub-tile 0 by cp.async into RES_BYTES of shared memory
  // at the start of the tile, sub-tile 1 into registers before the last wgmma wait
  static constexpr bool RES_PREFETCH = (BN == 128 && NSUB == 2 && NACC == 1 && TAPS == 9 && RC == 0);
  static constexpr int RES_BYTES = RES_PREFETCH ? 128 * BN * 2 : 0;
  static constexpr int B_STAGES_MAX = (BUDGET - A_STAGES * A_BYTES - RES_BYTES) / B_BYTES;
  static constexpr int B_STAGES = RC ? RC * TG : (B_STAGES_MAX > 8 ? 8 : B_STAGES_MAX);
  // release the stages of chunk c only once chunk c+1 is issued (one wgmma group in flight) when the weight ring can hold
  // two chunks; otherwise each weight stage is waited for and handed back right after its MMAs
  static constexpr bool LAG = RC || B_STAGES >= 2 * TG;
  static constexpr int ACOLS = NACC * BN;                                   // accumulator columns per sub-tile
  static constexpr int SMEM_BYTES = A_STAGES * A_BYTES + B_STAGES * B_BYTES + RES_BYTES + 1024;
  static_assert(NSUB * ACOLS <= 256, "register accumulator overflow");
  static_assert(B_STAGES >= 2, "not enough shared memory for the weight ring");
  static_assert(A_STAGES >= 2, "not enough shared memory for the halo ring");
  static_assert(SMEM_BYTES + 3584 <= 227 * 1024, "shared memory overflow (dynamic + static)");
};

// Sub-pixel layers: the (phase, tap) weight slices are stored view-major, the slices that read one halo view adjacent in their
// weight stage.  Accumulator slots are ordered p0, p1, p3, p2 (phase = oy*2 + ox).  Each slice is one N = BN wgmma into its
// slot's BN accumulator columns: every MMA writes a register range of the same shape that is either identical to or disjoint
// from any other's, so the MMAs of a whole K chunk chain without waits, like the taps of the 3x3 path.  (One wider wgmma per
// view over its adjacent slots reads each view once, but wgmmas of different N into overlapping columns must not be in flight
// together: that issue drained the tensor pipe after every view and ran the wav2lip ConvTs 2-4.5x slower, DESIGN.md.)
// {weight stage, halo view (row offset), first slot, first weight slice, slots}
struct SubpixelView {
  int stage, view, slot0, brow, nslots;
};
constexpr int subpixel_view(int vy, int vx) { return (vy + 1) * kHaloP + (vx + 1); }
template <int TAPS>
struct SubpixelTable;
// ConvT(k3, s2): stage 0: v00->p0,p1,p3 | stage 1: v01->p1,p3 ; v11->p3 | stage 2: v00->p2 ; v10->p3,p2  (ConvT halos start at the
// tile origin: view = dy*10 + dx)
template <>
struct SubpixelTable<9> {
  static constexpr int NV = 5;
  static constexpr SubpixelView v[NV] = {{0, 0, 0, 0, 3}, {1, 1, 1, 0, 2}, {1, kHaloP + 1, 2, 2, 1}, {2, 0, 3, 2, 1}, {2, kHaloP, 2, 0, 2}};
};
// Upsample(nearest 2x) + conv3x3: output phase (a, b) = 2x2 conv over the low-res halo, 16 (phase, view) slices in 4 stages
template <>
struct SubpixelTable<16> {
  static constexpr int NV = 10;
  static constexpr SubpixelView v[NV] = {{0, subpixel_view(0, 0), 0, 0, 4},
                                         {1, subpixel_view(-1, 0), 0, 0, 2},  {1, subpixel_view(0, 1), 1, 2, 2},
                                         {2, subpixel_view(1, 0), 2, 0, 2},   {2, subpixel_view(0, -1), 0, 2, 1}, {2, subpixel_view(0, -1), 3, 3, 1},
                                         {3, subpixel_view(-1, -1), 0, 0, 1}, {3, subpixel_view(-1, 1), 1, 1, 1}, {3, subpixel_view(1, 1), 2, 2, 1},
                                         {3, subpixel_view(1, -1), 3, 3, 1}};
};

// one view: weight slices BROW.. into accumulator slots SLOT0.., one N = BN wgmma each
template <int BN, int SLOT0, int BROW, int R, size_t... S>
__device__ __forceinline__ void subpixel_slots(float (&acc)[R], uint64_t a, uint32_t b_lo, uint32_t b_hi, std::index_sequence<S...>) {
  (wgmma_ss_at<BN, (SLOT0 + (int)S) * BN>(acc, a, wgmma_lohi(b_lo + (BROW + (uint32_t)S) * BN * 8u, b_hi), 1u), ...);
}

// the MMAs of weight stage j, K step k, views in table order.  j must be a compile-time constant after unrolling: the stage
// select then folds away and no branch sits between the MMAs.
template <int BN, int TAPS, int R, size_t... V>
__device__ __forceinline__ void subpixel_issue(float (&acc)[R], int j, int k, uint32_t a_lo0, uint32_t b_lo0, uint32_t a_hi, uint32_t b_hi,
                                               std::index_sequence<V...>) {
  (
      [&] {
        constexpr SubpixelView g = SubpixelTable<TAPS>::v[V];
        if (j == g.stage)
          subpixel_slots<BN, g.slot0, g.brow>(acc, wgmma_lohi(a_lo0 + g.view * 8u + k * 2u, a_hi), b_lo0 + k * 2u, b_hi,
                                              std::make_index_sequence<g.nslots>{});
      }(),
      ...);
}

// 4 x 4 transpose of 32-bit words across the four lanes of a quad (lane q's word j <-> lane j's word q), two xor-shuffle
// rounds.  Applied to the four channel-pair words of four 8-column blocks of one accumulator row, it turns "every lane holds
// channels 8i + 2q (+1) of blocks i" into "lane q holds all 8 channels of block q"; it is its own inverse.
__device__ __forceinline__ void quad_transpose(uint32_t (&x)[4], int lane) {
  const bool b2 = lane & 2, b1 = lane & 1;
  uint32_t s0 = __shfl_xor_sync(0xffffffffu, b2 ? x[0] : x[2], 2);
  uint32_t s1 = __shfl_xor_sync(0xffffffffu, b2 ? x[1] : x[3], 2);
  x[0] = b2 ? s0 : x[0];
  x[1] = b2 ? s1 : x[1];
  x[2] = b2 ? x[2] : s0;
  x[3] = b2 ? x[3] : s1;
  s0 = __shfl_xor_sync(0xffffffffu, b1 ? x[0] : x[1], 1);
  s1 = __shfl_xor_sync(0xffffffffu, b1 ? x[2] : x[3], 1);
  x[0] = b1 ? s0 : x[0];
  x[2] = b1 ? s1 : x[2];
  x[1] = b1 ? x[1] : s0;
  x[3] = b1 ? x[3] : s1;
}

// Instances that can take the residual from the halo (HaloParams::res_halo): 3x3 stride-1 convs with one accumulator slot.
// <128, 2, 1> is left out: its 128 accumulator floats, 64 residual words and the epilogue's GroupNorm partial sums do not fit
// the 232 consumer registers without spills, so it keeps reading the residual from global memory.
constexpr bool halo_res_smem_ok(int BN, int NSUB, int NACC, int TAPS) { return TAPS == 9 && NACC == 1 && BN * NSUB <= 128; }

// GRP: grouped GEMM mode (TAPS == 1 only): per-group M-tiles and weight slots, see HaloParams::group_slot
template <int BN, int NSUB, int NACC, int TAPS, int RC, bool GRP>
__global__ void __launch_bounds__(kHaloThreads, 1) conv_halo_wgmma_kernel(const __grid_constant__ HaloParams p) {
  static_assert(!GRP || TAPS == 1, "grouped weights exist in GEMM mode only");
  using C = HaloCfg<BN, NSUB, NACC, TAPS, RC>;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t a_full[C::A_STAGES], a_empty[C::A_STAGES];
  __shared__ __align__(8) uint64_t b_full[C::B_STAGES], b_empty[C::B_STAGES];
  __shared__ float head_sw[100];   // fused head: 3 x 32 weights + 3 biases
  // fused GroupNorm statistics: (sum, sum of squares) per (image, group) accumulated in SHARED memory across all tiles of this
  // persistent CTA and flushed with one global atomic per entry at the end
  constexpr int kGnSmem = (NACC == 1) ? 512 : 1;   // 8 images x 32 groups x (sum, sumsq); larger tables fall back to global atomics
  __shared__ float gn_acc[kGnSmem];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  constexpr bool kHeadOk = (BN == 32 && NACC == 1 && TAPS == 9);
  const bool gn_smem = NACC == 1 && p.gn_stats != nullptr && p.gn_images * p.gn_groups * 2 <= kGnSmem;
  if (gn_smem)
    for (int i = tid; i < p.gn_images * p.gn_groups * 2; i += kHaloThreads) gn_acc[i] = 0.f;
  constexpr bool kHaloMode = C::HALO;
  if (kHeadOk && p.head_out && tid < 99) head_sw[tid] = (tid < 96) ? p.head_w[tid] : p.head_b[tid - 96];
  const uint32_t smem0 = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t a_smem = smem0;
  const uint32_t b_smem = smem0 + C::A_STAGES * C::A_BYTES;
  const int chunks = (p.Cin + 63) / 64;
  const int kl_last = (p.Cin - 64 * (chunks - 1) + 15) / 16;   // K steps of 16 channels in the last chunk

  if (tid == 0) {
    for (int s = 0; s < C::A_STAGES; ++s) {
      mbar_init(smem_u32(&a_full[s]), 1);
      mbar_init(smem_u32(&a_empty[s]), 8);   // one arrival per consumer warp
    }
    for (int s = 0; s < C::B_STAGES; ++s) {
      mbar_init(smem_u32(&b_full[s]), 1);
      mbar_init(smem_u32(&b_empty[s]), 8);
    }
    mbar_fence_init();
    tma_prefetch_desc(&p.tm_in);
    tma_prefetch_desc(&p.tm_w);
  }
  __syncthreads();

  const int tiles_m = kHaloMode ? p.tiles_x * p.tiles_y * p.N : p.tiles_x;

  // PDL: the next kernel of the stream may start its own prologue now; resident weights (constants) are fetched before
  // this kernel waits for its predecessor, everything that touches activations comes after pdl_wait()
  pdl_launch_dependents();
  if (RC && warp == 8 && lane == 0) {
    // resident weights: every (chunk, tap-group) box once, all on b_full[0]
    mbar_arrive_expect_tx(smem_u32(&b_full[0]), RC * C::TG * C::B_BYTES);
    for (int c = 0; c < RC; ++c)
      for (int j = 0; j < C::TG; ++j)
        tma_load_3d(b_smem + (c * C::TG + j) * C::B_BYTES, &p.tm_w, smem_u32(&b_full[0]), c * 64, 0, j * C::TG);
  }
  pdl_wait();

  if (warp >= 8) {
    // =============================================================== TMA producer
    setmaxnreg_dec<kProducerRegs>();
    if (warp == 8 && lane == 0) {
      uint32_t ai = 0, bi = 0;  // running stage counters
      for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x) {
        const int nt = t / tiles_m;
        int mt = t - nt * tiles_m;
        int img = 0, y0 = 0, x0 = 0;
        int g_row = 0, g_slot = 0;   // grouped: first A row of the tile and the group's weight slot
        if constexpr (GRP) {
          const int g = mt / p.group_tiles;
          g_row = g * p.group_rows + (mt - g * p.group_tiles) * (128 * NSUB);
          g_slot = p.group_slot[g];
        }
        if (kHaloMode) {
          img = mt / (p.tiles_x * p.tiles_y);
          mt -= img * (p.tiles_x * p.tiles_y);
          const int ty = mt / p.tiles_x, tx = mt - ty * p.tiles_x;
          y0 = ty * (16 * NSUB) + p.halo_y0;
          x0 = tx * 8 + p.halo_x0;
        }
        for (int c = 0; c < chunks; ++c) {
          const uint32_t as = ai % C::A_STAGES;
          mbar_wait(smem_u32(&a_empty[as]), ((ai / C::A_STAGES) & 1u) ^ 1u);
          if (LTB_DIAG(8)) {
            mbar_arrive(smem_u32(&a_full[as]));
          } else {
            mbar_arrive_expect_tx(smem_u32(&a_full[as]), C::A_BYTES_RAW);
            if (C::S2) {
              // plane (rp, cp): rows of parity rp, columns of parity cp.  Odd planes start one plane-pixel early (input index 2*x0 - 1)
#pragma unroll
              for (int pl = 0; pl < 4; ++pl)
                tma_load_4d(a_smem + as * C::A_BYTES + pl * C::PLANE_BYTES, &p.tm_in, smem_u32(&a_full[as]), c * 64,
                            2 * (x0 + 1) - (pl & 1), 2 * (y0 + 1) - (pl >> 1), img);
            } else if (kHaloMode) tma_load_4d(a_smem + as * C::A_BYTES, &p.tm_in, smem_u32(&a_full[as]), c * 64, x0, y0, img);
            else if constexpr (GRP) tma_load_2d(a_smem + as * C::A_BYTES, &p.tm_in, smem_u32(&a_full[as]), c * 64, g_row);
            else tma_load_2d(a_smem + as * C::A_BYTES, &p.tm_in, smem_u32(&a_full[as]), c * 64, mt * (128 * NSUB));
          }
          ++ai;
          if (RC) continue;
          for (int j = 0; j < C::TG; ++j) {
            const uint32_t bs = bi % C::B_STAGES;
            mbar_wait(smem_u32(&b_empty[bs]), ((bi / C::B_STAGES) & 1u) ^ 1u);
            if (LTB_DIAG(16)) {
              mbar_arrive(smem_u32(&b_full[bs]));
              ++bi;
              continue;
            }
            mbar_arrive_expect_tx(smem_u32(&b_full[bs]), C::B_BYTES);
            if (kHaloMode) tma_load_3d(b_smem + bs * C::B_BYTES, &p.tm_w, smem_u32(&b_full[bs]), c * 64, nt * BN, j * C::TG);
            else if constexpr (GRP) tma_load_3d(b_smem + bs * C::B_BYTES, &p.tm_w, smem_u32(&b_full[bs]), c * 64, nt * BN, g_slot);
            else tma_load_2d(b_smem + bs * C::B_BYTES, &p.tm_w, smem_u32(&b_full[bs]), c * 64, nt * BN);
            ++bi;
          }
        }
      }
    }
  } else {
    // =============================================================== consumers: wgmma + epilogue
    setmaxnreg_inc<kConsumerRegs>();
    const int wg = warp >> 2, wq = warp & 3;
    const int cq = 2 * (lane & 3);
    constexpr uint32_t kAHi = wgmma_hi_128b(C::P * 128);   // SBO = halo pitch (1280 B) / 1024 B in GEMM mode
    constexpr uint32_t kBHi = wgmma_hi_128b(1024);
    // this warpgroup's first MMA row inside a sub-tile / plane: pixel row 8*wg (halo modes), row 64*wg (GEMM mode)
    constexpr uint32_t kRowsPerSub = C::HALO ? 16u * C::P : 128u;
    const uint32_t wg_off = (uint32_t)wg * (C::HALO ? 8u * C::P : 64u) * 8u;   // in 16-byte descriptor units
    // residual from the halo (p.res_halo): output channels [n0, n0 + BN) of a 3x3 conv whose residual is its own input are the
    // centre view (dy = dx = 1) of the halo stages of K chunks n0/64 (and n0/64 + 1 for BN = 128).  ldmatrix.x4 reads
    // matrices (row half hh, channel block i) = (0, i), (1, i), (0, i+1), (1, i+1): lanes 8k..8k+7 address rows 0..7 of matrix k,
    // and each lane receives its accumulator-fragment words rh[sub][hh][i] (row lane/4 + 8hh, channels 8i + cq (+1)).
    constexpr bool kResHalo = halo_res_smem_ok(BN, NSUB, NACC, TAPS);
    const int res_row = (8 * wg + 2 * wq + ((lane >> 3) & 1) + 1) * C::P + (lane & 7) + 1;   // halo row of MMA row (r % 8 = lane % 8)
    const int res_kb = lane >> 4;
    // halo modes: output (and residual) pixel of MMA row r of sub-tile `sub`, accumulator slot sl; ok = false past the map's edge
    auto halo_pix = [&](int img, int ty, int tx, int sub, int sl, int r, bool& ok) -> size_t {
      const int gy = ty * (16 * NSUB) + sub * 16 + wg * 8 + (r >> 3), gx = tx * 8 + (r & 7);
      ok = gy < p.GH && gx < p.GW;   // tiles may overhang small / odd-sized maps
      return ((size_t)img * p.OH + gy * p.osy + p.acc_oy[sl]) * p.OW + gx * p.osx + p.acc_ox[sl];
    };
    // RES_PREFETCH: sub-tile 0's residual, 16 bytes per (row half hh, 32-channel block m) of each consumer thread, laid out
    // [hh][m][thread] so that a warp's accesses are contiguous.  Each thread reads back only the slots it filled itself.
    const uint32_t res_buf = b_smem + C::B_STAGES * C::B_BYTES;
    if (RC) mbar_wait(smem_u32(&b_full[0]), 0);
    uint32_t ai = 0, bi = 0;
    for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x) {
      const int nt = t / tiles_m;
      int mt = t - nt * tiles_m;
      int img = 0, ty = 0, tx = 0;
      if (kHaloMode) {
        img = mt / (p.tiles_x * p.tiles_y);
        mt -= img * (p.tiles_x * p.tiles_y);
        ty = mt / p.tiles_x;
        tx = mt - ty * p.tiles_x;
      }
      const int n0 = nt * BN;
      const bool res_pf = C::RES_PREFETCH && p.res != nullptr && !LTB_DIAG(1);
      // the residual of MMA row r of sub-tile sub: 8 channels per 32-channel block, the lane's block of the row
      auto res_src = [&](int sub, int r, bool& ok) {
        const size_t px = halo_pix(img, ty, tx, sub, 0, r, ok);
        return reinterpret_cast<const uint4*>(p.res + (ok ? px : 0) * p.RCtot + p.rc_off + n0 + 8 * (lane & 3));
      };
      if constexpr (C::RES_PREFETCH) {
        if (res_pf) {   // the slots were last read in the previous tile's epilogue, by this thread, before its stores
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            bool ok;
            const uint4* src = res_src(0, wq * 16 + (lane >> 2) + 8 * hh, ok);
#pragma unroll
            for (int m = 0; m < BN / 32; ++m) cp_async16(res_buf + ((hh * (BN / 32) + m) * 256 + tid) * 16, src + 4 * m, ok ? 16u : 0u);
          }
          cp_async_commit();
        }
      }
      uint4 rpf[2][BN / 32];   // RES_PREFETCH: sub-tile 1's residual
      float acc[NSUB][C::ACOLS / 2];
#pragma unroll
      for (int s = 0; s < NSUB; ++s)
#pragma unroll
        for (int i = 0; i < C::ACOLS / 2; ++i) acc[s][i] = 0.f;
      uint32_t rh[NSUB][2][BN / 8];
      const int n0_res = (t / tiles_m) * BN;
      const int c_res = (kResHalo && p.res_halo) ? n0_res / 64 : chunks;   // chunks: no chunk holds it
      const int cb_res = (BN == 32) ? (n0_res & 63) >> 3 : 0;              // first 8-channel block of the tile in its chunk
      uint32_t pend_as = 0, pend_bs = 0;   // stages of the previous chunk (LAG mode), released once its wgmma group retired
      bool pend = false;
      // K chunk c, KL K steps of 16 channels per weight stage
      auto run_chunk = [&](int c, auto kl_t) {
        constexpr int KL = decltype(kl_t)::value;
        const uint32_t as = ai % C::A_STAGES;
        mbar_wait(smem_u32(&a_full[as]), (ai / C::A_STAGES) & 1u);
        if constexpr (kResHalo) {
          // read here, while this warp still holds the stage (it is handed back after this chunk's MMAs, or the next chunk's)
          if (c == c_res || (BN == 128 && c == c_res + 1)) {
            const bool hi = BN == 128 && c != c_res;
            const uint32_t rbase = a_smem + as * C::A_BYTES + res_row * 128;
#pragma unroll
            for (int s = 0; s < NSUB; ++s)
#pragma unroll
              for (int i = 0; i < BN / 8; i += 2) {
                if (BN == 128 && (i >= 8) != hi) continue;
                // 128B swizzle on a 1024-aligned stage: 16-byte chunk (channel / 8) XOR (halo row & 7); 16 * P rows per sub-tile
                // keep the row's phase
                const uint32_t chunk16 = (uint32_t)(((cb_res + i + res_kb) & 7) ^ (res_row & 7));
                ldmatrix_x4(rh[s][0][i], rh[s][1][i], rh[s][0][i + 1], rh[s][1][i + 1], rbase + s * (16 * C::P * 128) + chunk16 * 16);
              }
          }
        }
        const uint32_t a_lo0 = wgmma_lo(a_smem + as * C::A_BYTES) + wg_off;
        const uint32_t bs0 = bi % C::B_STAGES;
        // unrolled: a data-dependent branch around wgmma makes ptxas serialise the wgmma pipeline
#pragma unroll
        for (int j = 0; j < C::TG; ++j) {
          const uint32_t bs = RC ? (uint32_t)(c * C::TG + j) : (bi + j) % C::B_STAGES;
          if (!RC) mbar_wait(smem_u32(&b_full[bs]), ((bi + j) / C::B_STAGES) & 1u);
          const uint32_t b_lo0 = wgmma_lo(b_smem + bs * C::B_BYTES);
          if (!LTB_DIAG(4)) wgmma_fence();
#pragma unroll
          for (int k = 0; k < KL; ++k) {
            if (LTB_DIAG(4)) break;
            if constexpr (NACC == 1) {
#pragma unroll
              for (int tt = 0; tt < C::TG; ++tt) {
                // stride 2: tap (dy = j, dx = tt) reads plane (dy != 1, dx != 1) at view (dy == 2, dx == 2)
                const uint32_t aoff = C::S2 ? (uint32_t)(((j != 1) * 2 + (tt != 1)) * (C::PLANE_BYTES / 16) + ((j == 2) * C::P + (tt == 2)) * 8)
                                            : (kHaloMode ? (uint32_t)(j * C::P + tt) * 8u : 0u);
                const uint64_t bd = wgmma_lohi(b_lo0 + tt * (BN * 8) + k * 2, kBHi);
#pragma unroll
                for (int sub = 0; sub < NSUB; ++sub)
                  Wgmma<BN>::ss(acc[sub], wgmma_lohi(a_lo0 + aoff + sub * kRowsPerSub * 8 + k * 2, kAHi), bd, 1u);
              }
            } else {
              subpixel_issue<BN, TAPS>(acc[0], j, k, a_lo0, b_lo0, kAHi, kBHi, std::make_index_sequence<SubpixelTable<TAPS>::NV>{});
            }
          }
          if constexpr (!C::LAG) {   // the weight ring holds less than two chunks: hand each weight stage back as soon as it is read
            wgmma_commit();
            wgmma_wait<0>();
            __syncwarp();
            if (lane == 0) mbar_arrive(smem_u32(&b_empty[bs]));
          }
        }
        if (C::LAG) {
          wgmma_commit();
          wgmma_wait<1>();   // the group of chunk c-1 has retired: its stages go back to the producer
          if (pend) {
            __syncwarp();
            if (lane == 0) {
              mbar_arrive(smem_u32(&a_empty[pend_as]));
              if (!RC)
                for (int j = 0; j < C::TG; ++j) mbar_arrive(smem_u32(&b_empty[(pend_bs + j) % C::B_STAGES]));
            }
          }
          pend = true;
          pend_as = as;
          pend_bs = bs0;
        } else {
          __syncwarp();
          if (lane == 0) mbar_arrive(smem_u32(&a_empty[as]));
        }
        ++ai;
        if (!RC) bi += C::TG;
      };
      // A last chunk that holds at most 32 channels issues only its first two K steps: TMA zero-fills the rest of both operands,
      // whose products would add exact zeros.  It runs after the loop over the full chunks as a separate unrolled chunk body, so
      // that no branch sits between MMAs.  One such body, not one per step count: every extra body made the kernel's code larger
      // and the full-chunk layers slower (per-op events on an H100 80GB HBM3, 700 W limit: 2-5 us on the 128-channel and ConvT
      // layers of the wav2lip256 decoder with bodies for one, two and three steps), while two steps cover the 16- and 32-channel
      // remainders of wav2lip256 (L15/L16, L50, L53 and the audio encoder, all BN <= 64).  The BN = 128 instances, already the
      // largest (the two-step body took <128, 2, 1> from 6.7 k to 7.1 k SASS lines), keep four steps in every chunk.
      const bool ragged = BN <= 64 && kl_last <= 2;
#pragma unroll 1
      for (int c = 0; c < chunks - ragged; ++c) run_chunk(c, std::integral_constant<int, 4>{});
      if (ragged) run_chunk(chunks - 1, std::integral_constant<int, 2>{});
      if constexpr (C::RES_PREFETCH) {
        if (res_pf) {   // under the last chunk's MMAs
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            bool ok;
            const uint4* src = res_src(1, wq * 16 + (lane >> 2) + 8 * hh, ok);
#pragma unroll
            for (int m = 0; m < BN / 32; ++m) rpf[hh][m] = ok ? __ldcg(src + 4 * m) : make_uint4(0u, 0u, 0u, 0u);
          }
        }
      }
      wgmma_wait<0>();
      if (C::RES_PREFETCH && res_pf) cp_async_wait<0>();
#pragma unroll
      for (int s = 0; s < NSUB; ++s) wgmma_fence_regs(acc[s]);
      if (C::LAG && pend) {
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(smem_u32(&a_empty[pend_as]));
          if (!RC)
            for (int j = 0; j < C::TG; ++j) mbar_arrive(smem_u32(&b_empty[(pend_bs + j) % C::B_STAGES]));
        }
      }
      if (LTB_DIAG(2)) continue;

      // ---------------------------------------------------------- epilogue from the accumulator fragments
      const float* bias = p.bias;
      int g_tile = 0;   // grouped: this tile's group; its rows [g_tile * group_rows, (g_tile + 1) * group_rows) are the only ones written
      if constexpr (GRP) {
        g_tile = mt / p.group_tiles;
        bias += p.group_slot[g_tile] * p.bias_slot_stride;
      }
      const bool has_res = (p.res != nullptr) && !LTB_DIAG(1);
      const bool res_smem = kResHalo && has_res && p.res_halo;   // residual in rh, added in accumulator order
      const bool res_gmem = has_res && !res_smem;                // residual read from p.res after the quad transpose
      const bool head = kHeadOk && p.head_out != nullptr;
      float2 bb[BN / 8];
#pragma unroll
      for (int i = 0; i < BN / 8; ++i) bb[i] = __ldg(reinterpret_cast<const float2*>(bias + n0 + 8 * i + cq));
      const __half2 hmax = __floats2half2_rn(65504.f, 65504.f);
      const __half2 hlo = p.relu ? __floats2half2_rn(0.f, 0.f) : __floats2half2_rn(-65504.f, -65504.f);
      // (conv + bias) + residual, clamped: the same fp16 operation on either residual path
      auto add_res = [&](uint32_t v, uint32_t r) {
        const __half2 o = __hmin2(__hmax2(__hadd2(*reinterpret_cast<const __half2*>(&v), *reinterpret_cast<const __half2*>(&r)), hlo), hmax);
        return *reinterpret_cast<const uint32_t*>(&o);
      };
      // fused head: the lane's channel-pair words of its rows (sub, hh), row 2 sub + hh (unused rows of NSUB = 1 stay zero)
      uint32_t hrow[4][4] = {};
#pragma unroll
      for (int sub = 0; sub < NSUB; ++sub) {
        // GroupNorm partial sums of this warp's 16 rows, per 8-column block
        float gs[BN / 8], gq[BN / 8];
#pragma unroll
        for (int i = 0; i < BN / 8; ++i) gs[i] = gq[i] = 0.f;
#pragma unroll
        for (int sl = 0; sl < NACC; ++sl) {
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int r = wq * 16 + (lane >> 2) + 8 * hh;   // MMA row inside this warpgroup's 64
            size_t opix;
            bool row_ok;
            if (kHaloMode) {
              opix = halo_pix(img, ty, tx, sub, sl, r, row_ok);
            } else if constexpr (GRP) {
              // rows past the group's end belong to the next group, computed here with the wrong weights: never written
              const int lrow = (mt - g_tile * p.group_tiles) * (128 * NSUB) + sub * 128 + wg * 64 + r;
              opix = (size_t)g_tile * p.group_rows + lrow;
              row_ok = lrow < p.group_rows;
            } else {
              opix = (size_t)mt * (128 * NSUB) + sub * 128 + wg * 64 + r;   // GEMM mode: output row index
              row_ok = opix < (size_t)p.M;
            }
            // block 4m + (lane & 3) of this row: 8 channels, 16-byte aligned (conv_halo_supported)
            const size_t ocol = n0 + 8 * (lane & 3);
            uint4* optr = reinterpret_cast<uint4*>(p.out + opix * p.OCtot + p.oc_off + ocol);
            const uint4* rptr = res_gmem ? reinterpret_cast<const uint4*>(p.res + opix * p.RCtot + p.rc_off + ocol) : nullptr;
            __half2 oh[BN / 8];   // the row's values in accumulator order (lane holds channels 8i + cq (+1))
#pragma unroll
            for (int m = 0; m < BN / 32; ++m) {
              uint32_t v[4];
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const int i = 4 * m + j;
                const float f0 = acc[sub][sl * BN / 2 + 4 * i + 2 * hh] + bb[i].x;
                const float f1 = acc[sub][sl * BN / 2 + 4 * i + 2 * hh + 1] + bb[i].y;
                v[j] = (!has_res && p.relu) ? f32x2_to_f16x2_sat_relu(f0, f1) : f32x2_to_f16x2_sat(f0, f1);
                if constexpr (kResHalo)
                  if (res_smem) v[j] = add_res(v[j], rh[sub][hh][i]);
                oh[i] = *reinterpret_cast<const __half2*>(&v[j]);
              }
              if (!head || res_gmem) {
                quad_transpose(v, lane);
                if (res_gmem) {
                  uint4 r4 = make_uint4(0u, 0u, 0u, 0u);   // rows past the map's edge: zero, never stored
                  if constexpr (C::RES_PREFETCH) r4 = sub == 0 ? lds128(res_buf + ((hh * (BN / 32) + m) * 256 + tid) * 16) : rpf[hh][m];
                  else if (row_ok) r4 = __ldcg(rptr + 4 * m);
                  const uint32_t rv[4] = {r4.x, r4.y, r4.z, r4.w};
#pragma unroll
                  for (int j = 0; j < 4; ++j) v[j] = add_res(v[j], rv[j]);
                }
                if (row_ok && !head && !LTB_DIAG(1)) optr[4 * m] = make_uint4(v[0], v[1], v[2], v[3]);
                if (res_gmem && (p.gn_stats || head)) {   // the statistics and the head read the sums in accumulator order
                  quad_transpose(v, lane);
#pragma unroll
                  for (int j = 0; j < 4; ++j) oh[4 * m + j] = *reinterpret_cast<const __half2*>(&v[j]);
                }
              }
            }
            if (p.gn_stats && row_ok) {
#pragma unroll
              for (int i = 0; i < BN / 8; ++i) {
                const float2 f = __half22float2(oh[i]);
                gs[i] += f.x + f.y;
                gq[i] += f.x * f.x + f.y * f.y;
              }
            }
            if constexpr (kHeadOk)
#pragma unroll
              for (int i = 0; i < 4; ++i) hrow[2 * sub + hh][i] = *reinterpret_cast<const uint32_t*>(&oh[i]);
          }
        }
        // GEMM mode: a warp whose 16 rows all lie at or past M (the second sub-tile of a ragged last tile) has nothing to add, and
        // its image index would point one table past the end
        const size_t gn_row0 = (size_t)mt * (128 * NSUB) + sub * 128 + wg * 64 + wq * 16;
        if (p.gn_stats && (kHaloMode || gn_row0 < (size_t)p.M)) {
          int gimg = img;
          if (!kHaloMode) gimg = (int)(gn_row0 / (size_t)p.gn_hw);
          float* sbase = (gn_smem ? gn_acc : p.gn_stats) + (size_t)gimg * p.gn_groups * 2;
#pragma unroll
          for (int i = 0; i < BN / 8; ++i) {
            float a = gs[i], b = gq[i];
            // rows (lane / 4) always reduce; the column lanes reduce within a group: 4 channels = lane pairs
#pragma unroll
            for (int o = 4; o < 32; o <<= 1) {
              a += __shfl_xor_sync(0xffffffffu, a, o);
              b += __shfl_xor_sync(0xffffffffu, b, o);
            }
            a += __shfl_xor_sync(0xffffffffu, a, 1);
            b += __shfl_xor_sync(0xffffffffu, b, 1);
            if (p.gn_cpg >= 8) {
              a += __shfl_xor_sync(0xffffffffu, a, 2);
              b += __shfl_xor_sync(0xffffffffu, b, 2);
            }
            if (lane == 0 || (p.gn_cpg == 4 && lane == 2)) {
              const int g = (n0 + 8 * i + cq) / p.gn_cpg;
              atomicAdd(sbase + 2 * g, a);
              atomicAdd(sbase + 2 * g + 1, b);
            }
          }
        }
      }
      if constexpr (kHeadOk) {
        if (head) {
          // The four lanes of a quad share its 2 * NSUB rows and each holds channels 8i + 2(lane%4) (+1) of them.  A 4 x 4 word
          // transpose per 8-channel block i gives lane q all 32 channels of row q, and the lane computes the row's three outputs,
          // each summed in channel order (the order of w2l_head_kernel, so the fused head is bit-identical to the separate one).
          uint32_t hv[4][4];   // [src][i]: channels 8i + 2 src (+1) of row q
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            uint32_t x[4] = {hrow[0][i], hrow[1][i], hrow[2][i], hrow[3][i]};
            quad_transpose(x, lane);
#pragma unroll
            for (int src = 0; src < 4; ++src) hv[src][i] = x[src];
          }
          const int q = lane & 3;
          bool row_ok = false;
          const size_t opix = halo_pix(img, ty, tx, q >> 1, 0, wq * 16 + (lane >> 2) + 8 * (q & 1), row_ok);
          if (q < 2 * NSUB && row_ok) {
            float ha0 = head_sw[96], ha1 = head_sw[97], ha2 = head_sw[98];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
              for (int src = 0; src < 4; ++src) {
                const float2 f = __half22float2(*reinterpret_cast<__half2*>(&hv[src][i]));
                const int cc = 8 * i + 2 * src;
                ha0 = fmaf(f.x, head_sw[cc], ha0);
                ha0 = fmaf(f.y, head_sw[cc + 1], ha0);
                ha1 = fmaf(f.x, head_sw[32 + cc], ha1);
                ha1 = fmaf(f.y, head_sw[32 + cc + 1], ha1);
                ha2 = fmaf(f.x, head_sw[64 + cc], ha2);
                ha2 = fmaf(f.y, head_sw[64 + cc + 1], ha2);
              }
            float* o = p.head_out + opix * 3;
            o[0] = (1.f / (1.f + expf(-ha0))) * 255.f;
            o[1] = (1.f / (1.f + expf(-ha1))) * 255.f;
            o[2] = (1.f / (1.f + expf(-ha2))) * 255.f;
          }
        }
      }
    }
  }

  __syncthreads();
  if (gn_smem) {
    for (int i = tid; i < p.gn_images * p.gn_groups * 2; i += kHaloThreads) {
      const float v = gn_acc[i];
      if (v != 0.f) atomicAdd(p.gn_stats + i, v);
    }
  }
}

// ------------------------------------------------------------------------------------------------ host side
static bool is_convT(const ConvParams& p) {
  if (p.nphases != 4 || p.osy != 2 || p.osx != 2 || p.sy != 1 || p.sx != 1) return false;
  const int nt[4] = {1, 2, 2, 4};
  for (int i = 0; i < 4; ++i)
    if (p.ph[i].ntaps != nt[i]) return false;
  return p.IH == p.GH && p.IW == p.GW && p.OH == 2 * p.GH && p.OW == 2 * p.GW;
}

static bool is_conv3x3_s2(const ConvParams& p) {
  if (p.nphases != 1 || p.ph[0].ntaps != 9 || p.sy != 2 || p.sx != 2 || p.osy != 1 || p.osx != 1) return false;
  for (int t = 0; t < 9; ++t)
    if (p.ph[0].dy[t] != t / 3 - 1 || p.ph[0].dx[t] != t % 3 - 1) return false;
  return p.IH == 2 * p.GH && p.IW == 2 * p.GW && p.OH == p.GH && p.OW == p.GW;
}

static bool is_upconv(const ConvParams& p) {
  return p.upconv == 1 && p.nphases == 4 && p.osy == 2 && p.osx == 2 && p.sy == 1 && p.sx == 1 && p.IH == p.GH && p.IW == p.GW &&
         p.OH == 2 * p.GH && p.OW == 2 * p.GW;
}

static bool is_gemm(const ConvParams& p) {
  return p.nphases == 1 && p.ph[0].ntaps == 1 && p.ph[0].dy[0] == 0 && p.ph[0].dx[0] == 0 && p.sy == 1 && p.sx == 1 && p.osy == 1 &&
         p.osx == 1 && p.IH == p.GH && p.IW == p.GW && p.OH == p.GH && p.OW == p.GW;
}

static bool pick_cfg(const ConvParams& p, int* BN, int* NSUB, int* NACC);

bool conv_halo_supported(const ConvParams& p) {
  if (p.zbatch > 1) return false;   // the halo kernel runs one GEMM per launch
  // the epilogue writes the output (and reads the residual) 8 channels per 16-byte access
  if (!tma_slice_ok(p.out, p.OCtot, p.oc_off)) return false;
  if (p.res && !tma_slice_ok(p.res, p.RCtot, p.rc_off)) return false;
  // grouped weights: GEMM mode only (the weight map's slot stride must be 16-byte aligned); 3x3, stride-2, ConvT and upsample
  // layers go to the gather kernel
  if (p.group_slot && (!is_gemm(p) || (p.w_slot_stride * 2) % 16 != 0)) return false;
  if (is_gemm(p)) {
    // TMA GEMM: K-major rows with 16-byte aligned pitch; worth it from a few M tiles upwards
    return p.Cout % 32 == 0 && p.Cin % 8 == 0 && p.Cin >= 32 && (p.ICtot % 8) == 0 && (p.ic_off % 8) == 0 && (p.Ktot % 8) == 0 &&
           (p.ph[0].koff % 8) == 0 && p.M >= 512 && tma_encode_available();
  }
  if (is_conv3x3_s2(p)) {
    // parity-plane TMA path: worth it while the 16-row tiles are mostly full (the 8x8 / 4x4 output maps stay on the split-K gather
    // kernel) and a tile carries enough MMAs to hide the four plane loads behind two A stages.  Measured (profiles/r02l_per_op):
    // 64->128 @64->32: 18.5 -> 14.4 us, 128->256 @32->16: 22.5 -> 14.3 us, but 16->32 @256->128: 38.9 -> 64.1 us (nine K=16
    // instructions per 78 KB of zero-padded plane loads: latency bound) -> Cin >= 64 only.
    return p.Cout % 32 == 0 && p.Cin >= 64 && (p.ICtot % 8) == 0 && (p.ic_off % 8) == 0 && p.Ktot == 9 * p.Cin && p.GH >= 16 &&
           p.GW >= 8 && tma_encode_available();
  }
  if (is_upconv(p))
    return p.Cout % 64 == 0 && p.Cin >= 16 && (p.ICtot % 8) == 0 && (p.ic_off % 8) == 0 && p.Ktot == 16 * p.Cin && tma_encode_available();
  if (!(conv_is_3x3_same(p) || is_convT(p))) return false;
  // tiles of 16*NSUB x 8 pixels may overhang the map (TMA zero-fills the halo, the epilogue masks the stores): small maps
  // (8x8, 4x4 ...) waste MMA rows but still beat the latency-bound gather kernel
  if (p.Cout % 32 != 0 || p.Cin < 16) return false;
  if ((p.ICtot % 8) || (p.ic_off % 8) || (p.Ktot != 9 * p.Cin)) return false;
  if (p.GH % 16 != 0 || p.GW % 8 != 0) {
    // overhanging tiles burn MMA rows on pixels that do not exist: worth it only while the whole layer is a short chain
    // (w2l 512-channel 4x4 / 8x8 maps at batch 16: 1 wave x 8..16 K chunks); the 1280-channel 4x4 / 8x8 maps of the MuseTalk
    // UNet at batch 8 (2 waves x 20 chunks) stay on the split-K gather kernel, which measured faster there
    int BN, NSUB, NACC;
    if (!pick_cfg(p, &BN, &NSUB, &NACC)) return false;
    const long tiles = (long)p.N * ((p.GH + 16 * NSUB - 1) / (16 * NSUB)) * ((p.GW + 7) / 8) * (p.Cout / BN);
    const long waves = (tiles + kSms - 1) / kSms, chunks = (p.Cin + 63) / 64;
    if (waves * chunks > 16) return false;
  }
  return tma_encode_available();
}

// picks (BN, NSUB, NACC) ; returns false if unsupported
static bool pick_cfg(const ConvParams& p, int* BN, int* NSUB, int* NACC) {
  if (is_gemm(p)) {
    *NACC = 1;
    *BN = (p.Cout % 128 == 0) ? 128 : (p.Cout % 64 == 0) ? 64 : 32;
    auto tiles = [&](int bn, int nsub) { return (long)((p.M + 128 * nsub - 1) / (128 * nsub)) * (p.Cout / bn); };
    *NSUB = tiles(*BN, 2) >= kSms ? 2 : 1;
    while (*BN > 32 && tiles(*BN, *NSUB) < kSms - kSms / 8) *BN >>= 1;
    // 256 x 128 fp32 accumulators spill and unroll past the instruction cache in GEMM mode: 128-wide tiles take one sub-tile
    if (*BN == 128) *NSUB = 1;
    return true;
  }
  if (is_upconv(p)) {
    *NACC = 4;
    *NSUB = 1;
    *BN = 64;
    return true;
  }
  if (is_conv3x3_s2(p)) {
    *NACC = 1;
    *NSUB = 1;
    *BN = (p.Cout % 64 == 0) ? 64 : 32;
    return true;
  }
  const bool tr = is_convT(p);
  *NACC = tr ? 4 : 1;
  if (tr) {
    *NSUB = 1;
    // four phase accumulators of BN columns live in the registers of each consumer warpgroup: BN <= 64
    *BN = (p.Cout % 64 == 0) ? 64 : 32;
    return true;
  }
  // 3x3 conv: pick the (BN, NSUB) with the lowest modelled MMA time.  An M=128,K=16 step costs ~55 + 0.2*N cycles (the A
  // fetch dominates at small N), a tile issues ksteps*9*NSUB of them, the persistent grid walks ceil(tiles/SMs) waves;
  // ~800 cycles per tile for pipeline fill and the epilogue.
  const long ksteps = (p.Cin + 15) / 16;
  double best = 1e30;
  for (int bn : {128, 64, 32}) {
    if (p.Cout % bn) continue;
    for (int nsub : {2, 1}) {
      if (nsub == 2 && (p.GH % 32) != 0) continue;
      const long tiles = (long)p.N * ((p.GH + 16 * nsub - 1) / (16 * nsub)) * ((p.GW + 7) / 8) * (p.Cout / bn);
      const long waves = (tiles + kSms - 1) / kSms;
      const double tile = (double)ksteps * 9 * nsub * (55.0 + 0.2 * bn) + 800.0;
      // single-wave launches cannot overlap their epilogue with the next tile's loads
      const double epi = (waves == 1) ? 40.0 * nsub * bn : 0.0;
      const double cost = waves * tile + epi;
      if (cost < best * 0.9) {   // prefer the earlier (wider) candidate unless the model predicts a clear (>10 %) win
        best = cost;
        *BN = bn;
        *NSUB = nsub;
      }
    }
  }
  return best < 1e30;
}

int conv_halo_make_plan(const ConvParams& p, const __half* w_tap_major, HaloPlan* out) {
  if (!conv_halo_supported(p)) return 1;
  HaloParams& h = out->hp;
  std::memset(&h, 0, sizeof(h));
  out->grouped = false;
  int BN, NSUB, NACC;
  if (!pick_cfg(p, &BN, &NSUB, &NACC)) return 1;
  out->BN = BN;
  out->NSUB = NSUB;
  out->NACC = NACC;
  const bool up = is_upconv(p);
  const bool s2 = is_conv3x3_s2(p);
  const bool tr = NACC == 4 && !up;
  const bool gemm = is_gemm(p);
  out->TAPS = gemm ? 1 : (up ? 16 : (s2 ? 10 : 9));
  if (gemm) {
    // A: 2-D (K, rows) ; B: 2-D (K, Cout) over the layer's own K-major weight rows
    cuuint64_t dims[2] = {(cuuint64_t)p.Cin, (cuuint64_t)p.M};
    cuuint64_t strides[1] = {(cuuint64_t)p.ICtot * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)(128 * NSUB)};
    if (!encode_tmap_f16(&h.tm_in, 2, p.in + p.ic_off, dims, strides, box)) return 2;
    // grouped: 3-D (K, Cout, slot) over the whole bank, one slot per box
    cuuint64_t wdims[3] = {(cuuint64_t)p.Cin, (cuuint64_t)p.Cout, (cuuint64_t)p.slots};
    cuuint64_t wstrides[2] = {(cuuint64_t)p.Ktot * 2, (cuuint64_t)p.w_slot_stride * 2};
    cuuint32_t wbox[3] = {64, (cuuint32_t)BN, 1};
    if (!encode_tmap_f16(&h.tm_w, p.group_slot ? 3 : 2, p.w + p.ph[0].koff, wdims, wstrides, wbox)) return 2;
  } else {
    cuuint32_t box[4] = {64, (cuuint32_t)kHaloP, (cuuint32_t)(16 * NSUB + 2), 1};
    if (s2) {   // one parity plane per load: 9 x (16*NSUB + 1) pixels picked with traversal stride 2 (box extent 2n - 1)
      box[1] = 2 * 9 - 1;
      box[2] = 2 * (16 * NSUB + 1) - 1;
    }
    if (!encode_nhwc_f16(&h.tm_in, p.in + p.ic_off, p.Cin, p.IW, p.IH, p.N, p.ICtot, box, s2 ? 2 : 1)) return 2;
  }
  // weights: 3-D (k = Cin, n = Cout, tap = 9) view of the tap-major copy [9][Cout][Cin]
  if (up) {
    // 16 view-major slices [16][Cout][Cin], four per weight stage
    cuuint64_t dims[3] = {(cuuint64_t)p.Cin, (cuuint64_t)p.Cout, 16};
    cuuint64_t strides[2] = {(cuuint64_t)p.Cin * 2, (cuuint64_t)p.Cout * p.Cin * 2};
    cuuint32_t box[3] = {64, (cuuint32_t)BN, 4};
    if (!encode_tmap_f16(&h.tm_w, 3, w_tap_major, dims, strides, box)) return 2;
  } else if (!gemm) {
    cuuint64_t dims[3] = {(cuuint64_t)p.Cin, (cuuint64_t)p.Cout, 9};
    cuuint64_t strides[2] = {(cuuint64_t)p.Cin * 2, (cuuint64_t)p.Cout * p.Cin * 2};
    cuuint32_t box[3] = {64, (cuuint32_t)BN, 3};
    if (!encode_tmap_f16(&h.tm_w, 3, w_tap_major, dims, strides, box)) return 2;
  }
  h.out = p.out;
  h.res = p.res;
  h.bias = p.bias;
  h.N = p.N;
  h.M = p.M;
  h.Cin = p.Cin;
  h.gn_stats = nullptr;
#ifdef LTB_HALO_DIAG
  if (const char* e = std::getenv("LTB_HALO_DIAG")) h.dbg = std::atoi(e);
#endif
  h.OCtot = p.OCtot;
  h.oc_off = p.oc_off;
  h.RCtot = p.RCtot;
  h.rc_off = p.rc_off;
  h.OH = p.OH;
  h.OW = p.OW;
  h.GH = p.GH;
  h.GW = p.GW;
  h.osy = p.osy;
  h.osx = p.osx;
  h.relu = p.relu;
  // the residual is exactly the input slice the halo tiles hold (the wav2lip residual blocks): channels [n0, n0 + BN) of the
  // tile's centre view
  h.res_halo = halo_res_smem_ok(BN, NSUB, NACC, out->TAPS) && p.res != nullptr && p.res == p.in && p.Cin == p.Cout &&
               p.rc_off == p.ic_off && p.RCtot == p.ICtot;
  h.halo_y0 = tr ? 0 : -1;
  h.halo_x0 = tr ? 0 : -1;
  if (up || tr) {
    // accumulator slots p0, p1, p3, p2 (phase index = oy*2 + ox), see SubpixelTable
    const int slot_phase[4] = {0, 1, 3, 2};
    for (int sl = 0; sl < 4; ++sl) {
      h.acc_oy[sl] = p.ph[slot_phase[sl]].ooy;
      h.acc_ox[sl] = p.ph[slot_phase[sl]].oox;
    }
  } else {
    h.acc_oy[0] = p.ph[0].ooy;
    h.acc_ox[0] = p.ph[0].oox;
  }
  h.tiles_n = p.Cout / BN;
  if (gemm) {
    h.halo_y0 = h.halo_x0 = 0;
    h.tiles_x = (p.M + 128 * NSUB - 1) / (128 * NSUB);
    if (p.group_slot) {
      out->grouped = true;
      h.group_slot = p.group_slot;
      h.group_rows = p.group_images * p.GH * p.GW;
      h.group_tiles = (h.group_rows + 128 * NSUB - 1) / (128 * NSUB);
      h.bias_slot_stride = p.bias_slot_stride;
      h.tiles_x = (p.N / p.group_images) * h.group_tiles;
    }
    h.tiles_y = 1;
    h.total_tiles = h.tiles_x * h.tiles_n;
    return 0;
  }
  h.tiles_x = (p.GW + 7) / 8;
  h.tiles_y = (p.GH + 16 * NSUB - 1) / (16 * NSUB);
  h.total_tiles = h.tiles_x * h.tiles_y * p.N * h.tiles_n;
  return 0;
}

template <int BN, int NSUB, int NACC, int TAPS = 9, int RC = 0, bool GRP = false>
static cudaError_t launch_cfg(const HaloPlan& pl, int sms, cudaStream_t st) {
  using C = HaloCfg<BN, NSUB, NACC, TAPS, RC>;
  static SmemConfigOnce once;
  if (cudaError_t e = once.ensure(conv_halo_wgmma_kernel<BN, NSUB, NACC, TAPS, RC, GRP>, C::SMEM_BYTES); e != cudaSuccess) return e;
  const int grid = pl.hp.total_tiles < sms ? pl.hp.total_tiles : sms;
  return launch_kernel_pdl(conv_halo_wgmma_kernel<BN, NSUB, NACC, TAPS, RC, GRP>, dim3(grid), dim3(kHaloThreads), C::SMEM_BYTES, st, pl.hp);
}

// weights-resident variants: 3x3 / ConvT layers with a single N tile, at least two tiles per SM and one or two K chunks of
// weights (the variants that fit next to the halo ring)
int conv_halo_resident_chunks(const HaloPlan& pl, int sms) {
  if (pl.TAPS != 9 || pl.hp.tiles_n != 1 || pl.hp.total_tiles < 2 * sms) return 0;
  const int key = pl.BN * 100 + pl.NSUB * 10 + pl.NACC;
  const int chunks = (pl.hp.Cin + 63) / 64;
  if (chunks == 1 && (key == 6421 || key == 3221 || key == 6414 || key == 3214)) return 1;
  if (chunks == 2 && (key == 3221 || key == 6414 || key == 3214)) return 2;
  return 0;
}

cudaError_t launch_conv_halo(const HaloPlan& pl, cudaStream_t st) {
  const int sms = device_sms();
  if (pl.TAPS == 10) {
    if (pl.NSUB != 1 || pl.NACC != 1) return cudaErrorInvalidValue;
    return pl.BN == 64 ? launch_cfg<64, 1, 1, 10>(pl, sms, st) : (pl.BN == 32 ? launch_cfg<32, 1, 1, 10>(pl, sms, st) : cudaErrorInvalidValue);
  }
  if (pl.TAPS == 16) return (pl.BN == 64 && pl.NSUB == 1 && pl.NACC == 4) ? launch_cfg<64, 1, 4, 16>(pl, sms, st) : cudaErrorInvalidValue;
  const int key = pl.BN * 100 + pl.NSUB * 10 + pl.NACC;
  if (pl.TAPS == 1 && pl.grouped) {
    switch (key) {
      case 12811: return launch_cfg<128, 1, 1, 1, 0, true>(pl, sms, st);
      case 6421: return launch_cfg<64, 2, 1, 1, 0, true>(pl, sms, st);
      case 6411: return launch_cfg<64, 1, 1, 1, 0, true>(pl, sms, st);
      case 3221: return launch_cfg<32, 2, 1, 1, 0, true>(pl, sms, st);
      case 3211: return launch_cfg<32, 1, 1, 1, 0, true>(pl, sms, st);
    }
    return cudaErrorInvalidValue;
  }
  if (pl.TAPS == 1) {
    switch (key) {
      case 12811: return launch_cfg<128, 1, 1, 1>(pl, sms, st);
      case 6421: return launch_cfg<64, 2, 1, 1>(pl, sms, st);
      case 6411: return launch_cfg<64, 1, 1, 1>(pl, sms, st);
      case 3221: return launch_cfg<32, 2, 1, 1>(pl, sms, st);
      case 3211: return launch_cfg<32, 1, 1, 1>(pl, sms, st);
    }
    return cudaErrorInvalidValue;
  }
  // weights-resident variants (single N tile, whole weight set in shared memory)
  switch (conv_halo_resident_chunks(pl, sms) * 100000 + key) {
    case 106421: return launch_cfg<64, 2, 1, 9, 1>(pl, sms, st);
    case 103221: return launch_cfg<32, 2, 1, 9, 1>(pl, sms, st);
    case 203221: return launch_cfg<32, 2, 1, 9, 2>(pl, sms, st);
    case 206414: return launch_cfg<64, 1, 4, 9, 2>(pl, sms, st);
    case 106414: return launch_cfg<64, 1, 4, 9, 1>(pl, sms, st);
    case 103214: return launch_cfg<32, 1, 4, 9, 1>(pl, sms, st);
    case 203214: return launch_cfg<32, 1, 4, 9, 2>(pl, sms, st);
  }
  switch (key) {
    case 12821: return launch_cfg<128, 2, 1>(pl, sms, st);
    case 12811: return launch_cfg<128, 1, 1>(pl, sms, st);
    case 6421: return launch_cfg<64, 2, 1>(pl, sms, st);
    case 6411: return launch_cfg<64, 1, 1>(pl, sms, st);
    case 3221: return launch_cfg<32, 2, 1>(pl, sms, st);
    case 3211: return launch_cfg<32, 1, 1>(pl, sms, st);
    case 6414: return launch_cfg<64, 1, 4>(pl, sms, st);
    case 3214: return launch_cfg<32, 1, 4>(pl, sms, st);
  }
  return cudaErrorInvalidValue;
}

// can the epilogue of this plan accumulate GroupNorm statistics of its output?  (power-of-two channels per group >= 4,
// whole 16-row groups inside one image)
bool conv_halo_gn_fusable(const HaloPlan& pl, int cout_total, int groups, int hw) {
  if (pl.NACC != 1 || groups <= 0 || cout_total % groups) return false;
  const int cpg = cout_total / groups;
  if (cpg < 4 || (cpg & (cpg - 1))) return false;
  if (pl.TAPS == 1 && (hw % 128) != 0) return false;
  return true;
}

// [Cout][ntaps][Cin] -> [ntaps][Cout][Cin] (one-off, at model load)
__global__ void w_tap_major_kernel(const __half* __restrict__ w, __half* __restrict__ wt, int cout, int cin, int ntaps) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)cout * ntaps * cin;
  if (i >= total) return;
  const int ci = (int)(i % cin);
  const int tap = (int)((i / cin) % ntaps);
  const int co = (int)(i / ((size_t)cin * ntaps));
  wt[((size_t)tap * cout + co) * cin + ci] = w[i];
}

cudaError_t launch_w_tap_major(const __half* w, __half* wt, int cout, int cin, cudaStream_t st, int ntaps) {
  const size_t total = (size_t)cout * ntaps * cin;
  w_tap_major_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(w, wt, cout, cin, ntaps);
  return cudaGetLastError();
}

// phase-major slice s (p0:(0,0) | p1:(0,0),(0,1) | p2:(0,0),(1,0) | p3:(0,0),(0,1),(1,0),(1,1)) -> view-major position
__global__ void w_tap_major_convT_kernel(const __half* __restrict__ w, __half* __restrict__ wt, int cout, int cin) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)cout * 9 * cin;
  if (i >= total) return;
  const int ci = (int)(i % cin);
  const int tap = (int)((i / cin) % 9);
  const int co = (int)(i / ((size_t)cin * 9));
  // new order: [v00p0, v00p1, v00p3 | v01p1, v01p3, v11p3 | v10p3, v10p2, v00p2] = old slices [0,1,5 | 2,6,8 | 7,4,3]
  const int pos_of_old[9] = {0, 1, 3, 8, 7, 2, 4, 6, 5};
  wt[((size_t)pos_of_old[tap] * cout + co) * cin + ci] = w[i];
}

cudaError_t launch_w_tap_major_convT(const __half* w, __half* wt, int cout, int cin, cudaStream_t st) {
  const size_t total = (size_t)cout * 9 * cin;
  w_tap_major_convT_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(w, wt, cout, cin);
  return cudaGetLastError();
}

}  // namespace ltb
