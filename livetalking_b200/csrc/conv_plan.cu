// Conv planning (conv_plan.h): ConvParams construction, kernel choice, epilogue fusions, launch, and the stand-alone conv
// test hook of the C ABI (ltb_conv2d_f16).  Host code only.
#include <cstring>
#include <string>
#include <vector>

#include "../../include/ltb200.h"
#include "conv_plan.h"
#include "conv_tma.h"
#include "ltb_internal.h"

namespace ltb {

// ConvTranspose2d(k=3, s=2, p=1, op=1): out[2g+a] gathers (d=0,k=1) for a=0 and (d=0,k=2),(d=+1,k=0) for a=1.
static const int kTd[2][2] = {{0, 0}, {0, 1}};
static const int kTk[2][2] = {{1, 0}, {2, 0}};
static const int kTn[2] = {1, 2};
// nearest 2x upsample + 3x3 p1 conv: out[2g+a] reads low-resolution rows {-1, 0} for a=0 and {0, +1} for a=1
static const int kUd[2][2] = {{-1, 0}, {0, 1}};

ConvParams conv_params(ConvMode mode, int N, ConvSlice in, int IH, int IW, int Cin, ConvSlice out, int OH, int OW, int Cout,
                       ConvSlice res, const __half* w, int Ktot, int w_koff, const float* bias, bool relu, ConvTaps taps) {
  ConvParams p;
  std::memset(&p, 0, sizeof(p));
  p.in = in.p;
  p.N = N;
  p.IH = IH;
  p.IW = IW;
  p.ICtot = in.Ctot;
  p.ic_off = in.off;
  p.Cin = Cin;
  p.sy = p.sx = 1;
  p.out = const_cast<__half*>(out.p);
  p.OH = OH;
  p.OW = OW;
  p.OCtot = out.Ctot;
  p.oc_off = out.off;
  p.osy = p.osx = 1;
  p.Cout = Cout;
  p.res = res.p;
  p.RCtot = res.Ctot;
  p.rc_off = res.off;
  p.w = w;
  p.Ktot = Ktot;
  p.bias = bias;
  p.relu = relu ? 1 : 0;
  if (mode == ConvMode::Dense) {
    p.sy = taps.sy;
    p.sx = taps.sx;
    p.GH = OH;
    p.GW = OW;
    p.nphases = 1;
    ConvPhase& ph = p.ph[0];
    ph.ntaps = taps.KH * taps.KW;
    ph.koff = w_koff;
    for (int kh = 0; kh < taps.KH; ++kh)
      for (int kw = 0; kw < taps.KW; ++kw) {
        ph.dy[kh * taps.KW + kw] = (signed char)(kh - taps.pad_t);
        ph.dx[kh * taps.KW + kw] = (signed char)(kw - taps.pad_l);
      }
  } else {
    // four sub-pixel phases over the input grid: phase (a, b) writes output pixels (2y + a, 2x + b)
    const bool up = mode == ConvMode::Upsample2x;
    p.GH = IH;
    p.GW = IW;
    p.osy = p.osx = 2;
    p.nphases = 4;
    p.upconv = up ? 1 : 0;
    int koff = w_koff;
    for (int a = 0; a < 2; ++a)
      for (int b = 0; b < 2; ++b) {
        ConvPhase& ph = p.ph[a * 2 + b];
        const int na = up ? 2 : kTn[a], nb = up ? 2 : kTn[b];
        ph.ntaps = na * nb;
        ph.koff = koff;
        ph.ooy = a;
        ph.oox = b;
        for (int i = 0; i < na; ++i)
          for (int j = 0; j < nb; ++j) {
            ph.dy[i * nb + j] = (signed char)(up ? kUd[a][i] : kTd[a][i]);
            ph.dx[i * nb + j] = (signed char)(up ? kUd[b][j] : kTd[b][j]);
          }
        koff += ph.ntaps * Cin;
      }
  }
  p.M = N * p.GH * p.GW;
  return p;
}

int conv_plan(const ConvParams& p, const __half* w_tap, ConvPath path, ConvPlan* out) {
  out->p = p;
  out->kernel = ConvKernel::Gather;
  if (p.group_slot) {
    if (p.group_images < 1 || p.N % p.group_images || p.slots < 1 || p.w_slot_stride < 0 || p.bias_slot_stride < 0)
      return LTB_FAIL("conv: grouped weights need N divisible by group_images >= 1, slots >= 1 and non-negative slot strides");
    if (p.zbatch > 1 || p.upconv) return LTB_FAIL("conv: grouped weights cannot be combined with zbatch or the fused upsample");
  }
  if (path == ConvPath::Gather) return 0;
  if (path == ConvPath::Auto && conv_smallmap_supported(p)) {
    if (conv_smallmap_make_plan(p, &out->sp) != 0) return LTB_FAIL("conv: small-map plan / tensor map creation failed");
    out->kernel = ConvKernel::Smallmap;
    return 0;
  }
  if (w_tap && conv_pingpong_supported(p)) {
    if (conv_pingpong_make_plan(p, w_tap, &out->pp) != 0) return LTB_FAIL("conv: ping-pong plan / tensor map creation failed");
    out->kernel = ConvKernel::Pingpong;
    return 0;
  }
  if (w_tap && conv_rowpair_supported(p)) {
    if (conv_rowpair_make_plan(p, w_tap, &out->rp) != 0) return LTB_FAIL("conv: row-pair plan / tensor map creation failed");
    out->kernel = ConvKernel::Rowpair;
    return 0;
  }
  const bool gemm = p.nphases == 1 && p.ph[0].ntaps == 1;   // the halo kernel's GEMM mode reads the K-major rows
  if (!((w_tap || gemm) && conv_halo_supported(p))) {
    if (path == ConvPath::Auto) return 0;
    return LTB_FAIL("conv: the halo kernel cannot run " + std::to_string(p.N) + "x" + std::to_string(p.IH) + "x" + std::to_string(p.IW) +
                    "x" + std::to_string(p.Cin) + " -> " + std::to_string(p.OH) + "x" + std::to_string(p.OW) + "x" + std::to_string(p.Cout) +
                    (w_tap || gemm ? "" : " without tap-major weights"));
  }
  if (conv_halo_make_plan(p, w_tap, &out->hp) != 0) return LTB_FAIL("conv: halo plan / tensor map creation failed");
  out->kernel = ConvKernel::Halo;
  return 0;
}

cudaError_t conv_launch(const ConvPlan& pl, cudaStream_t st, float* splitk_ws, size_t ws_floats) {
  switch (pl.kernel) {
    case ConvKernel::Gather: return launch_conv_gather(pl.p, st, splitk_ws, ws_floats);
    case ConvKernel::Halo: return launch_conv_halo(pl.hp, st);
    case ConvKernel::Pingpong: return launch_conv_pingpong(pl.pp, st);
    case ConvKernel::Rowpair: return launch_conv_rowpair(pl.rp, st);
    case ConvKernel::Smallmap: return launch_conv_smallmap(pl.sp, st);
  }
  return cudaErrorInvalidValue;
}

bool conv_plan_variant(const ConvPlan& pl, bool have_ws, size_t ws_floats, ltb_conv_variant* out) {
  std::memset(out, 0, sizeof(*out));
  out->kernel = int(pl.kernel);
  out->grouped = pl.p.group_slot != nullptr;
  switch (pl.kernel) {
    case ConvKernel::Pingpong:   // one instance: 3x3, 64 output channels, one 128-pixel tile per warpgroup, resident weights
      out->taps = 9;
      out->bn = 64;
      out->nsub = 1;
      out->nacc = 1;
      out->resident_chunks = 1;
      out->res_halo = 1;
      return true;
    case ConvKernel::Rowpair:   // one instance: 3x3, 32 output channels, two resident K chunks
      out->taps = 9;
      out->bn = 32;
      out->nsub = 1;
      out->nacc = 1;
      out->resident_chunks = 2;
      return true;
    case ConvKernel::Smallmap:   // 128 output channels per CTA, 64-channel K steps, ksplit CTAs of a cluster per output tile
      for (int i = 0; i < pl.p.nphases; ++i) out->taps += pl.p.ph[i].ntaps;
      out->bn = 128;
      out->kb = 64;
      out->ksplit = pl.sp.ksplit;
      return true;
    case ConvKernel::Halo:
      out->taps = pl.hp.TAPS;
      out->bn = pl.hp.BN;
      out->nsub = pl.hp.NSUB;
      out->nacc = pl.hp.NACC;
      out->resident_chunks = conv_halo_resident_chunks(pl.hp, device_sms());
      out->res_halo = pl.hp.hp.res_halo;
      return true;
    case ConvKernel::Gather:
      break;
  }
  int ksplit = 0;
  if (!conv_gather_pick(pl.p, have_ws, ws_floats, &out->bn, &out->kb, &ksplit)) return false;
  out->ksplit = ksplit > 1 ? ksplit : 1;
  return true;
}

bool conv_plan_fuse_gn_stats(ConvPlan* pl, float* stats, int groups, int hw) {
  const ConvParams& p = pl->p;
  if (pl->kernel != ConvKernel::Halo || pl->hp.grouped || p.oc_off != 0 || p.OCtot != p.Cout ||
      !conv_halo_gn_fusable(pl->hp, p.Cout, groups, hw))
    return false;
  HaloParams& h = pl->hp.hp;
  h.gn_stats = stats;
  h.gn_groups = groups;
  h.gn_cpg = p.Cout / groups;
  h.gn_hw = hw;
  h.gn_images = p.M / hw;
  return true;
}

bool conv_plan_fuse_head(ConvPlan* pl, const float* w, const float* b, float* out) {
  if (pl->kernel == ConvKernel::Rowpair) {
    pl->rp.head_w = w;
    pl->rp.head_b = b;
    pl->rp.head_out = out;
    return true;
  }
  if (pl->kernel != ConvKernel::Halo || pl->hp.grouped || pl->hp.BN != 32 || pl->p.Cout != 32) return false;
  pl->hp.hp.head_w = w;
  pl->hp.hp.head_b = b;
  pl->hp.hp.head_out = out;
  return true;
}

// host-side packing of PyTorch-layout float weights into the kernels' K-major fp16 rows (ltb_conv2d_f16 only; the model
// path receives rows already packed by livetalking_b200/w2l_pack.py, which follows the same order)
static void pack_conv_w(const float* w, int cout, int cin, int KH, int KW, std::vector<__half>& out) {
  out.resize((size_t)cout * KH * KW * cin);
  for (int co = 0; co < cout; ++co)
    for (int kh = 0; kh < KH; ++kh)
      for (int kw = 0; kw < KW; ++kw)
        for (int ci = 0; ci < cin; ++ci)
          out[((size_t)co * KH * KW + kh * KW + kw) * cin + ci] = __float2half(w[(((size_t)co * cin + ci) * KH + kh) * KW + kw]);
}
static void pack_convT_w(const float* w, int cin, int cout, std::vector<__half>& out) {
  out.resize((size_t)cout * 9 * cin);
  for (int co = 0; co < cout; ++co) {
    size_t k = 0;
    for (int a = 0; a < 2; ++a)
      for (int b = 0; b < 2; ++b)
        for (int i = 0; i < kTn[a]; ++i)
          for (int j = 0; j < kTn[b]; ++j) {
            const int kh = kTk[a][i], kw = kTk[b][j];
            for (int ci = 0; ci < cin; ++ci, ++k)
              out[(size_t)co * 9 * cin + k] = __float2half(w[(((size_t)ci * cout + co) * 3 + kh) * 3 + kw]);
          }
  }
}

}  // namespace ltb

using namespace ltb;

static int conv2d_f16_impl(const ltb_conv_desc* d, const void* in_f16, const float* w_f32, const float* bias_f32,
                           const void* res_f16, void* out_f16, int reps, float* ms_out) {
  if (!d || !in_f16 || !w_f32 || !bias_f32 || !out_f16) return LTB_FAIL("null argument");
  if (d->has_res && !res_f16) return LTB_FAIL("has_res set but res is null");
  int OH, OW, Ktot;
  std::vector<__half> wp;
  if (d->transposed) {
    if (d->KH != 3 || d->KW != 3) return LTB_FAIL("transposed conv: only k=3,s=2,p=1,op=1");
    OH = d->IH * 2;
    OW = d->IW * 2;
    Ktot = 9 * d->Cin;
    pack_convT_w(w_f32, d->Cin, d->Cout, wp);
  } else {
    if (d->KH * d->KW > kMaxTaps) return LTB_FAIL("kernel too large");
    OH = conv_out_dim(d->IH, d->KH, d->sy, d->pad);
    OW = conv_out_dim(d->IW, d->KW, d->sx, d->pad);
    Ktot = d->KH * d->KW * d->Cin;
    pack_conv_w(w_f32, d->Cout, d->Cin, d->KH, d->KW, wp);
  }
  if (OH <= 0 || OW <= 0) return LTB_FAIL("empty output");
  const size_t in_b = (size_t)d->N * d->IH * d->IW * d->Cin * 2, out_b = (size_t)d->N * OH * OW * d->Cout * 2;
  __half *din = nullptr, *dout = nullptr, *dw = nullptr, *dres = nullptr, *dwt = nullptr;
  float* dbias = nullptr;
  float* dws = nullptr;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  int rc = 0;
  auto cleanup = [&]() {
    cudaFree(din);
    cudaFree(dout);
    cudaFree(dw);
    cudaFree(dres);
    cudaFree(dwt);
    cudaFree(dws);
    cudaFree(dbias);
    if (e0) cudaEventDestroy(e0);
    if (e1) cudaEventDestroy(e1);
  };
#define CK(x)                                                             \
  do {                                                                    \
    cudaError_t _e = (x);                                                 \
    if (_e != cudaSuccess) {                                              \
      rc = LTB_FAIL(std::string(#x) + ": " + cudaGetErrorString(_e));     \
      cleanup();                                                          \
      return rc;                                                          \
    }                                                                     \
  } while (0)
  CK(cudaMalloc(&din, in_b));
  CK(cudaMalloc(&dout, out_b));
  CK(cudaMalloc(&dw, wp.size() * 2));
  CK(cudaMalloc(&dbias, (size_t)d->Cout * 4));
  CK(cudaMemcpy(din, in_f16, in_b, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dw, wp.data(), wp.size() * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dbias, bias_f32, (size_t)d->Cout * 4, cudaMemcpyHostToDevice));
  CK(cudaMemset(dout, 0xFF, out_b));  // NaN pattern: unwritten outputs are caught by the test
  if (d->has_res) {
    CK(cudaMalloc(&dres, out_b));
    CK(cudaMemcpy(dres, res_f16, out_b, cudaMemcpyHostToDevice));
  }
  if (d->KH == 3 && d->KW == 3) {   // the halo kernel reads 3x3 and ConvT weights from a tap-major copy
    CK(cudaMalloc(&dwt, wp.size() * 2));
    CK(d->transposed ? launch_w_tap_major_convT(dw, dwt, d->Cout, d->Cin, nullptr) : launch_w_tap_major(dw, dwt, d->Cout, d->Cin, nullptr));
  }
  const ConvParams p = conv_params(d->transposed ? ConvMode::Transposed : ConvMode::Dense, d->N, {din, d->Cin, 0}, d->IH, d->IW, d->Cin,
                                   {dout, d->Cout, 0}, OH, OW, d->Cout, d->has_res ? ConvSlice{dres, d->Cout, 0} : ConvSlice{}, dw, Ktot, 0,
                                   dbias, d->relu != 0, {d->KH, d->KW, d->sy, d->sx, d->pad, d->pad});
  const ConvPath path = d->force_path == 1 ? ConvPath::Gather : d->force_path == 2 ? ConvPath::Halo : ConvPath::Auto;
  ConvPlan pl;
  if (conv_plan(p, dwt, path, &pl)) {
    cleanup();
    return 1;
  }
  const size_t ws_floats = pl.kernel == ConvKernel::Gather ? (size_t)1 << 22 : 0;   // split-K workspace of the gather kernel
  if (ws_floats) {
    CK(cudaMalloc(&dws, ws_floats * sizeof(float)));
    CK(cudaMemset(dws, 0, ws_floats * sizeof(float)));
  }
  CK(conv_launch(pl, nullptr, dws, ws_floats));
  if (reps > 0) {   // back-to-back launches of the same plan between two events (kernel development aid)
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    for (int i = 0; i < 3; ++i) CK(conv_launch(pl, nullptr, dws, ws_floats));
    CK(cudaEventRecord(e0, nullptr));
    for (int i = 0; i < reps; ++i) CK(conv_launch(pl, nullptr, dws, ws_floats));
    CK(cudaEventRecord(e1, nullptr));
    CK(cudaEventSynchronize(e1));
    CK(cudaEventElapsedTime(ms_out, e0, e1));
    *ms_out /= reps;
  }
  CK(cudaDeviceSynchronize());
  CK(cudaMemcpy(out_f16, dout, out_b, cudaMemcpyDeviceToHost));
#undef CK
  cleanup();
  return 0;
}

extern "C" {

int ltb_conv2d_f16(const ltb_conv_desc* d, const void* in_f16, const float* w_f32, const float* bias_f32,
                   const void* res_f16, void* out_f16) {
  return conv2d_f16_impl(d, in_f16, w_f32, bias_f32, res_f16, out_f16, 0, nullptr);
}

int ltb_conv2d_f16_timed(const ltb_conv_desc* d, const void* in_f16, const float* w_f32, const float* bias_f32,
                         const void* res_f16, void* out_f16, int reps, float* ms_per_launch) {
  if (reps < 1 || !ms_per_launch) return LTB_FAIL("conv2d_f16_timed: reps >= 1 and a result pointer are required");
  return conv2d_f16_impl(d, in_f16, w_f32, bias_f32, res_f16, out_f16, reps, ms_per_launch);
}

}  // extern "C"
