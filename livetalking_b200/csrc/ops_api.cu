// Generic device-op layer of the C ABI (include/ltb200.h, "ltb_ctx / ltb_op_*"): the MuseTalk networks (diffusers
// UNet2DConditionModel / AutoencoderKL and the Whisper encoder — third-party graphs the reference only wraps,
// avatars/musetalk/models/{unet,vae}.py, avatars/musetalk/whisper/audio2feature.py) are assembled by the Python host
// code out of these operators, captured ONCE into a CUDA graph and replayed per step.  Every op is asynchronous on the
// context's stream; device memory is owned by the context.
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/ltb200.h"
#include "conv_plan.h"
#include "ltb_internal.h"
#include "ops.h"

using namespace ltb;

struct ltb_ctx {
  int device = 0;
  cudaStream_t st = nullptr;
  std::mutex mu;                // guards `allocs` (a model ctx is shared by every session thread that uploads / frees)
  std::vector<void*> allocs;
  float* zero_bias = nullptr;   // 16384 zeros (bias of bias-free GEMMs)
  float* gn_ws = nullptr;       // GroupNorm statistics workspace
  float* splitk_ws = nullptr;   // fp32 split-K workspace (zero between uses)
  long long launches = 0;
  bool capturing = false;
  long long capture_launches = 0;
};
struct ltb_graph {
  cudaGraph_t g = nullptr;
  cudaGraphExec_t exec = nullptr;
  long long launches = 0;
};

// the calling thread may be a fresh render / inference / process thread whose current device is 0
#define LTB_CTX_ENTER(c)                                                                          \
  do {                                                                                            \
    int _cur = -1;                                                                                \
    if (cudaGetDevice(&_cur) != cudaSuccess || _cur != (c)->device) LTB_CUDA(cudaSetDevice((c)->device)); \
  } while (0)

static const int kZeroBias = 16384;
static const int kGnWsFloats = 64 * 64 * 2;
static const size_t kSplitKWsFloats = (size_t)16 << 20;  // ksplit * M * Cout floats

extern "C" {

int ltb_ctx_create(ltb_ctx** out) {
  if (!out) return LTB_FAIL("null argument");
  auto* c = new ltb_ctx();
  cudaError_t e = cudaGetDevice(&c->device);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&c->st, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void**>(&c->zero_bias), kZeroBias * sizeof(float));
  if (e == cudaSuccess) e = cudaMemset(c->zero_bias, 0, kZeroBias * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void**>(&c->gn_ws), kGnWsFloats * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void**>(&c->splitk_ws), kSplitKWsFloats * sizeof(float));
  if (e == cudaSuccess) e = cudaMemset(c->splitk_ws, 0, kSplitKWsFloats * sizeof(float));
  if (e != cudaSuccess) {
    delete c;
    return LTB_FAIL(std::string("ctx create: ") + cudaGetErrorString(e));
  }
  *out = c;
  return 0;
}

int ltb_ctx_destroy(ltb_ctx* c) {
  if (!c) return 0;
  cudaSetDevice(c->device);
  cudaStreamSynchronize(c->st);
  for (void* p : c->allocs) cudaFree(p);
  cudaFree(c->zero_bias);
  cudaFree(c->gn_ws);
  cudaFree(c->splitk_ws);
  cudaStreamDestroy(c->st);
  delete c;
  return 0;
}

int ltb_ctx_stream(ltb_ctx* c, void** stream) {
  if (!c || !stream) return LTB_FAIL("null argument");
  LTB_CTX_ENTER(c);
  *stream = static_cast<void*>(c->st);
  return 0;
}
int ltb_ctx_sync(ltb_ctx* c) {
  if (!c) return LTB_FAIL("null ctx");
  LTB_CTX_ENTER(c);
  LTB_CUDA(cudaStreamSynchronize(c->st));
  return 0;
}
int ltb_ctx_launch_count(ltb_ctx* c, long long* n) {
  if (!c || !n) return LTB_FAIL("null argument");
  LTB_CTX_ENTER(c);
  *n = c->launches;
  return 0;
}

int ltb_dev_alloc(ltb_ctx* c, size_t bytes, int zero, void** dptr) {
  if (!c || !dptr) return LTB_FAIL("null argument");
  LTB_CTX_ENTER(c);
  void* p = nullptr;
  LTB_CUDA(cudaMalloc(&p, bytes ? bytes : 16));
  if (zero) LTB_CUDA(cudaMemset(p, 0, bytes ? bytes : 16));
  {
    std::lock_guard<std::mutex> lk(c->mu);
    c->allocs.push_back(p);
  }
  *dptr = p;
  return 0;
}
int ltb_dev_free(ltb_ctx* c, void* dptr) {
  if (!c || !dptr) return 0;
  LTB_CTX_ENTER(c);
  {
    std::lock_guard<std::mutex> lk(c->mu);
    size_t i = 0;
    while (i < c->allocs.size() && c->allocs[i] != dptr) ++i;
    if (i == c->allocs.size()) return LTB_FAIL("dev_free: pointer not owned by this context");
    c->allocs.erase(c->allocs.begin() + i);
  }
  cudaFree(dptr);
  return 0;
}
int ltb_h2d(ltb_ctx* c, void* dst_dev, const void* src_host, size_t bytes, int sync) {
  if (!c) return LTB_FAIL("null ctx");
  LTB_CTX_ENTER(c);
  LTB_CUDA(cudaMemcpyAsync(dst_dev, src_host, bytes, cudaMemcpyHostToDevice, c->st));
  if (sync) LTB_CUDA(cudaStreamSynchronize(c->st));
  return 0;
}
int ltb_d2h(ltb_ctx* c, void* dst_host, const void* src_dev, size_t bytes, int sync) {
  if (!c) return LTB_FAIL("null ctx");
  LTB_CTX_ENTER(c);
  LTB_CUDA(cudaMemcpyAsync(dst_host, src_dev, bytes, cudaMemcpyDeviceToHost, c->st));
  if (sync) LTB_CUDA(cudaStreamSynchronize(c->st));
  return 0;
}
int ltb_d2d(ltb_ctx* c, void* dst_dev, const void* src_dev, size_t bytes) {
  if (!c || !dst_dev || !src_dev) return LTB_FAIL("d2d: null argument");
  LTB_CTX_ENTER(c);
  LTB_CUDA(cudaMemcpyAsync(dst_dev, src_dev, bytes, cudaMemcpyDeviceToDevice, c->st));
  return 0;
}
int ltb_set_i32(ltb_ctx* c, void* dptr, int value) {
  if (!c || !dptr) return LTB_FAIL("null argument");
  LTB_CTX_ENTER(c);
  LTB_CUDA(launch_set_int(static_cast<int*>(dptr), value, c->st));
  c->launches += 1;
  return 0;
}

// ---- graph capture ------------------------------------------------------------------------------
int ltb_capture_begin(ltb_ctx* c) {
  if (!c) return LTB_FAIL("null ctx");
  LTB_CTX_ENTER(c);
  if (c->capturing) return LTB_FAIL("already capturing");
  LTB_CUDA(cudaStreamBeginCapture(c->st, cudaStreamCaptureModeThreadLocal));
  c->capturing = true;
  c->capture_launches = c->launches;
  return 0;
}
int ltb_capture_end(ltb_ctx* c, ltb_graph** out) {
  if (!c || !out) return LTB_FAIL("null argument");
  LTB_CTX_ENTER(c);
  if (!c->capturing) return LTB_FAIL("not capturing");
  c->capturing = false;
  auto* g = new ltb_graph();
  cudaError_t e = cudaStreamEndCapture(c->st, &g->g);
  if (e == cudaSuccess) e = cudaGraphInstantiate(&g->exec, g->g, 0);
  if (e != cudaSuccess) {
    if (g->g) cudaGraphDestroy(g->g);
    delete g;
    return LTB_FAIL(std::string("graph capture/instantiate: ") + cudaGetErrorString(e));
  }
  g->launches = c->launches - c->capture_launches;
  c->launches = c->capture_launches;  // captured launches did not execute
  *out = g;
  return 0;
}
int ltb_graph_launch(ltb_ctx* c, ltb_graph* g) {
  if (!c || !g) return LTB_FAIL("null argument");
  LTB_CTX_ENTER(c);
  LTB_CUDA(cudaGraphLaunch(g->exec, c->st));
  c->launches += g->launches;
  return 0;
}
int ltb_graph_destroy(ltb_graph* g) {
  if (!g) return 0;
  if (g->exec) cudaGraphExecDestroy(g->exec);
  if (g->g) cudaGraphDestroy(g->g);
  delete g;
  return 0;
}

}  // extern "C"

// ---- ops ----------------------------------------------------------------------------------------

// argument checks and planning of ltb_op_conv2d, shared with ltb_op_conv2d_plan.  Returns 0, or 1 with the reason set.
static int conv2d_plan(ltb_ctx* c, const ltb_conv_op* d, ConvPlan* pl) {
  if (!d->in || !d->w || !d->out) return LTB_FAIL("conv2d: null argument");
  if (d->KH * d->KW > kMaxTaps) return LTB_FAIL("conv2d: kernel too large");
  if (d->Cout > kZeroBias && !d->bias) return LTB_FAIL("conv2d: Cout too large for the implicit zero bias");
  if (d->upsample2x && (d->KH != 3 || d->KW != 3 || d->sy != 1 || d->sx != 1 || d->pad_t != 1 || d->pad_l != 1 || d->OH != 2 * d->IH ||
                        d->OW != 2 * d->IW || d->Ktot != 16 * d->Cin || !d->w_tap || d->zbatch > 1))
    return LTB_FAIL("conv2d: upsample2x needs a 3x3 s1 p1 conv, OH = 2*IH, OW = 2*IW and the 16-slice weights");
  if (d->transposed && (d->upsample2x || d->KH != 3 || d->KW != 3 || d->OH != 2 * d->IH || d->OW != 2 * d->IW || d->Ktot != 9 * d->Cin ||
                        d->zbatch > 1))
    return LTB_FAIL("conv2d: transposed needs a 3x3 kernel, OH = 2*IH, OW = 2*IW, Ktot = 9*Cin and no upsample2x or zbatch");
  const ConvMode mode = d->upsample2x ? ConvMode::Upsample2x : d->transposed ? ConvMode::Transposed : ConvMode::Dense;
  ConvParams p = conv_params(mode, d->N,
                             {static_cast<const __half*>(d->in), d->ICtot, d->ic_off}, d->IH, d->IW, d->Cin,
                             {static_cast<const __half*>(d->out), d->OCtot, d->oc_off}, d->OH, d->OW, d->Cout,
                             {static_cast<const __half*>(d->res), d->RCtot, d->rc_off}, static_cast<const __half*>(d->w), d->Ktot,
                             d->w_koff, d->bias ? d->bias : c->zero_bias, d->relu != 0, {d->KH, d->KW, d->sy, d->sx, d->pad_t, d->pad_l});
  p.zbatch = d->zbatch;
  p.zdiv = d->zdiv > 0 ? d->zdiv : 1;
  p.in_zo = d->in_zo;
  p.in_zi = d->in_zi;
  p.w_zo = d->w_zo;
  p.w_zi = d->w_zi;
  p.out_zo = d->out_zo;
  p.out_zi = d->out_zi;
  p.smallmap = d->smallmap;
  if (d->group_slot) {
    if (d->gn_stats) return LTB_FAIL("conv2d: grouped weights cannot produce GroupNorm statistics");
    p.group_slot = static_cast<const int*>(d->group_slot);
    p.group_images = d->group_images;
    p.slots = d->slots;
    p.w_slot_stride = d->w_slot_stride;
    p.bias_slot_stride = d->bias_slot_stride;
  }
  // the fused upsample exists on the halo kernel only
  const ConvPath path = d->upsample2x ? ConvPath::Halo : d->no_halo == 1 ? ConvPath::Gather : d->no_halo == 2 ? ConvPath::Halo : ConvPath::Auto;
  return conv_plan(p, static_cast<const __half*>(d->w_tap), path, pl);
}

extern "C" {

int ltb_op_conv2d(ltb_ctx* c, const ltb_conv_op* d) {
  if (!c || !d) return LTB_FAIL("conv2d: null argument");
  LTB_CTX_ENTER(c);
  ConvPlan pl;
  if (conv2d_plan(c, d, &pl)) return 1;
  pdl_set_enabled(pdl_default());   // the calling thread may have run a w2l profiling pass with PDL off
  const ConvParams& p = pl.p;
  const bool want_stats = d->gn_stats != nullptr && d->gn_groups > 0 && d->gn_hw > 0 && (p.M % d->gn_hw) == 0 && d->zbatch <= 1;
  float* stats = static_cast<float*>(d->gn_stats);
  const bool stats_fused = want_stats && conv_plan_fuse_gn_stats(&pl, stats, d->gn_groups, d->gn_hw);
  if (stats_fused) LTB_CUDA(cudaMemsetAsync(stats, 0, (size_t)(p.M / d->gn_hw) * d->gn_groups * 2 * sizeof(float), c->st));
  cudaError_t e = conv_launch(pl, c->st, c->splitk_ws, kSplitKWsFloats);
  if (e != cudaSuccess) return LTB_FAIL(std::string("conv2d launch: ") + cudaGetErrorString(e));
  c->launches += 1;
  if (want_stats && !stats_fused) {
    // fallback: separate statistics pass over the freshly written output
    e = launch_gn_stats(static_cast<const __half*>(d->out), p.M / d->gn_hw, d->gn_hw, d->Cout, d->OCtot, d->oc_off, d->gn_groups, stats,
                        c->st);
    if (e != cudaSuccess) return LTB_FAIL(std::string("conv2d gn_stats: ") + cudaGetErrorString(e));
    c->launches += 1;
  }
  return 0;
}

int ltb_op_conv2d_plan(ltb_ctx* c, const ltb_conv_op* d, ltb_conv_variant* out) {
  if (!c || !d || !out) return LTB_FAIL("conv2d_plan: null argument");
  LTB_CTX_ENTER(c);
  ConvPlan pl;
  if (conv2d_plan(c, d, &pl)) return 1;
  if (!conv_plan_variant(pl, c->splitk_ws != nullptr, kSplitKWsFloats, out)) return LTB_FAIL("conv2d_plan: no kernel instance runs this geometry");
  return 0;
}

int ltb_op_w_tap_major(ltb_ctx* c, const void* w, void* wt, int cout, int cin) {
  if (!c || !w || !wt) return LTB_FAIL("null argument");
  LTB_CTX_ENTER(c);
  LTB_CUDA(launch_w_tap_major(static_cast<const __half*>(w), static_cast<__half*>(wt), cout, cin, c->st));
  c->launches += 1;
  return 0;
}

int ltb_op_groupnorm(ltb_ctx* c, const void* x, int N, int HW, int C, int Ctot, int c_off, int groups, float eps, const float* gamma,
                     const float* beta, int silu, void* out, int OCtot, int oc_off) {
  if (!c || !x || !out || !gamma || !beta) return LTB_FAIL("groupnorm: null argument");
  LTB_CTX_ENTER(c);
  if ((size_t)N * groups * 2 > (size_t)kGnWsFloats) return LTB_FAIL("groupnorm: batch too large for the statistics workspace");
  cudaError_t e = launch_groupnorm(static_cast<const __half*>(x), N, HW, C, Ctot, c_off, groups, eps, gamma, beta, silu,
                                   static_cast<__half*>(out), OCtot, oc_off, c->gn_ws, c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("groupnorm: ") + cudaGetErrorString(e));
  c->launches += 2;
  return 0;
}
int ltb_op_groupnorm_apply(ltb_ctx* c, const void* x, int N, int HW, int C, int Ctot, int c_off, int groups, float eps, const void* stats,
                           const float* gamma, const float* beta, int silu, void* out, int OCtot, int oc_off) {
  if (!c || !x || !out || !gamma || !beta || !stats) return LTB_FAIL("groupnorm_apply: null argument");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_gn_apply(static_cast<const __half*>(x), N, HW, C, Ctot, c_off, groups, eps, static_cast<const float*>(stats), gamma,
                                  beta, silu, static_cast<__half*>(out), OCtot, oc_off, c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("groupnorm_apply: ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_layernorm(ltb_ctx* c, const void* x, int rows, int C, float eps, const float* gamma, const float* beta, void* out) {
  if (!c || !x || !out) return LTB_FAIL("layernorm: null argument");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_layernorm(static_cast<const __half*>(x), rows, C, eps, gamma, beta, static_cast<__half*>(out), c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("layernorm: ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_softmax(ltb_ctx* c, const void* x, int rows, int cols, int ld, int valid, float scale, void* out) {
  if (!c || !x || !out) return LTB_FAIL("softmax: null argument");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_softmax(static_cast<const __half*>(x), rows, cols, ld, valid, scale, static_cast<__half*>(out), c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("softmax: ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_geglu(ltb_ctx* c, const void* h, long long rows, int H, void* out) {
  if (!c || !h || !out) return LTB_FAIL("geglu: null argument");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_geglu(static_cast<const __half*>(h), (size_t)rows, H, static_cast<__half*>(out), c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("geglu: ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_eltwise(ltb_ctx* c, const void* x, const void* y, long long n, long long period, int act, void* out) {
  if (!c || !x || !out) return LTB_FAIL("eltwise: null argument");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_eltwise(static_cast<const __half*>(x), static_cast<const __half*>(y), (size_t)n, (size_t)period, act,
                                 static_cast<__half*>(out), c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("eltwise: ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_upsample2x(ltb_ctx* c, const void* x, int N, int H, int W, int C, void* out) {
  if (!c || !x || !out) return LTB_FAIL("upsample2x: null argument");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_upsample2x(static_cast<const __half*>(x), N, H, W, C, static_cast<__half*>(out), c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("upsample2x: ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_copy_channels(ltb_ctx* c, const void* src, long long rows, int C, int SCtot, int sc_off, void* dst, int DCtot, int dc_off) {
  if (!c || !src || !dst) return LTB_FAIL("copy_channels: null argument");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_copy_channels(static_cast<const __half*>(src), (size_t)rows, C, SCtot, sc_off, static_cast<__half*>(dst), DCtot,
                                       dc_off, c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("copy_channels: ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_transpose_heads(ltb_ctx* c, const void* v, int B, int n_keys, int Ctot, int c_off, int heads, int d, int n_pad, void* vt) {
  if (!c || !v || !vt) return LTB_FAIL("transpose_heads: null argument");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_transpose_heads(static_cast<const __half*>(v), B, n_keys, Ctot, c_off, heads, d, n_pad, static_cast<__half*>(vt),
                                         c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("transpose_heads: ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_attention(ltb_ctx* c, const void* q, int q_pitch, const void* k, int kv_pitch, int kv_rows, const void* vt, int n_pad, int B, int heads,
                     int nq, int valid, int d, float scale, void* out, int out_pitch) {
  if (!c || !q || !k || !vt || !out) return LTB_FAIL("attention: null argument");
  if (!attn_fused_supported(d, q_pitch, kv_pitch, n_pad)) return LTB_FAIL("attention: unsupported head dim / pitch (d % 16 == 0, d <= 160, pitches % 8 == 0)");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_attn_fused(static_cast<const __half*>(q), q_pitch, static_cast<const __half*>(k), kv_pitch, kv_rows,
                                    static_cast<const __half*>(vt), n_pad, B, heads, nq, valid, d, scale, static_cast<__half*>(out), out_pitch, c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("attention: ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
// ---- UltraLight / HuBERT ops (SURVEY 8 row f4)
int ltb_op_dwconv3x3(ltb_ctx* c, const void* x, int N, int IH, int IW, int ICtot, int ic_off, int C, const void* w_tap, const float* bias, int stride,
                     int relu, void* out, int OCtot, int oc_off) {
  if (!c || !x || !w_tap || !bias || !out) return LTB_FAIL("dwconv3x3: null argument");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_dwconv3x3(static_cast<const __half*>(x), N, IH, IW, ICtot, ic_off, C, static_cast<const __half*>(w_tap), bias, stride, relu,
                                   static_cast<__half*>(out), OCtot, oc_off, c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("dwconv3x3 (C, pitches, offsets % 8 == 0; stride 1 | 2): ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_dwconv3x3_grouped(ltb_ctx* c, const void* x, int N, int IH, int IW, int ICtot, int ic_off, int C, const void* w_tap, const float* bias,
                             int stride, int relu, void* out, int OCtot, int oc_off, const int* group_slot, int group_images, long long w_slot_stride,
                             long long bias_slot_stride) {
  if (!c || !x || !w_tap || !bias || !out || !group_slot) return LTB_FAIL("dwconv3x3_grouped: null argument");
  LTB_CTX_ENTER(c);
  const WeightGroups grp{group_slot, group_images, w_slot_stride, bias_slot_stride};
  cudaError_t e = launch_dwconv3x3(static_cast<const __half*>(x), N, IH, IW, ICtot, ic_off, C, static_cast<const __half*>(w_tap), bias, stride, relu,
                                   static_cast<__half*>(out), OCtot, oc_off, c->st, &grp);
  if (e != cudaSuccess)
    return LTB_FAIL(std::string("dwconv3x3_grouped (C, pitches, offsets, w stride % 8 == 0; bias stride % 4 == 0; N % group_images == 0): ") +
                    cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_upsample_bilinear2x(ltb_ctx* c, const void* x, int N, int H, int W, int ICtot, int ic_off, int C, void* out, int OCtot, int oc_off) {
  if (!c || !x || !out) return LTB_FAIL("upsample_bilinear2x: null argument");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_upsample_bilinear2x(static_cast<const __half*>(x), N, H, W, ICtot, ic_off, C, static_cast<__half*>(out), OCtot, oc_off, c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("upsample_bilinear2x: ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_ul_prep(ltb_ctx* c, const void* faces_u8, int nf, const void* d_index, int B, void* out) {
  if (!c || !faces_u8 || !d_index || !out || nf < 1 || B < 1) return LTB_FAIL("ul_prep: bad argument");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_ul_prep(static_cast<const uint8_t*>(faces_u8), nf, static_cast<const int*>(d_index), B, static_cast<__half*>(out), c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("ul_prep: ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_ul_prep_grouped(ltb_ctx* c, const void* groups_dev, int group_images, int B, void* out) {
  static_assert(sizeof(UlPrepGroup) == sizeof(ltb_ul_prep_group), "ltb_ul_prep_group layout");
  if (!c || !groups_dev || !out || B < 1) return LTB_FAIL("ul_prep_grouped: bad argument");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_ul_prep_grouped(static_cast<const UlPrepGroup*>(groups_dev), group_images, B, static_cast<__half*>(out), c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("ul_prep_grouped (B % group_images == 0): ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_head_sigmoid255_grouped(ltb_ctx* c, const void* x, const float* w3x32, const float* b3, long long npix, float* pred, int hw,
                                   const int* group_slot, int group_images, long long w_slot_stride, long long bias_slot_stride) {
  if (!c || !x || !w3x32 || !b3 || !pred || !group_slot) return LTB_FAIL("head_sigmoid255_grouped: null argument");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_head_grouped(static_cast<const __half*>(x), w3x32, b3, pred, (int)npix, hw,
                                      WeightGroups{group_slot, group_images, w_slot_stride, bias_slot_stride}, c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("head_sigmoid255_grouped (hw % 256 == 0, whole groups): ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_head_sigmoid255(ltb_ctx* c, const void* x, const float* w3x32, const float* b3, long long npix, float* pred) {
  if (!c || !x || !w3x32 || !b3 || !pred) return LTB_FAIL("head_sigmoid255: null argument");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_w2l_head(static_cast<const __half*>(x), w3x32, b3, pred, (int)npix, c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("head_sigmoid255: ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_ul_paste(ltb_ctx* c, const void* frames, const void* faces, const void* coords, const float* pred, void* out, int nf, int H, int W,
                    int index, int explicit_idx, int slot0, int count) {
  if (!c || !frames || !faces || !coords || !pred || !out || nf < 1 || count < 1) return LTB_FAIL("ul_paste: bad argument");
  if (explicit_idx >= nf) return LTB_FAIL("ul_paste: frame index out of range");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_ul_paste(static_cast<const uint8_t*>(frames), static_cast<const uint8_t*>(faces), static_cast<const int*>(coords), pred,
                                  static_cast<uint8_t*>(out), nf, H, W, index, explicit_idx, slot0, count, c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("ul_paste: ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_hubert_conv0_grouped(ltb_ctx* c, const float* pcm, int G, int n, const float* w, const float* bias, int C, float* stats, void* out) {
  if (!c || !pcm || !w || !stats || !out) return LTB_FAIL("hubert_conv0: null argument");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_hubert_conv0(pcm, G, n, w, bias, C, stats, static_cast<__half*>(out), c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("hubert_conv0 (n >= 10, 1 <= G <= 65535): ") + cudaGetErrorString(e));
  c->launches += 2;
  return 0;
}
int ltb_op_hubert_pos_conv_grouped(ltb_ctx* c, const void* h, int G, int T, int D, int groups, int K, const void* w, const float* bias, void* out) {
  if (!c || !h || !w || !bias || !out) return LTB_FAIL("hubert_pos_conv: null argument");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_hubert_pos_conv(static_cast<const __half*>(h), G, T, D, groups, K, static_cast<const __half*>(w), bias,
                                         static_cast<__half*>(out), c->st);
  if (e != cudaSuccess)
    return LTB_FAIL(std::string("hubert_pos_conv (K = 128, D / groups = 64, out != h, 1 <= G <= 65535): ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_hubert_slice_grouped(ltb_ctx* c, const void* hidden, int G, int Tc, int T, int D, int B, int R, float start, float mult, int win_l,
                                float* out_f32, void* out_nhwc) {
  if (!c || !hidden || (!out_f32 && !out_nhwc)) return LTB_FAIL("hubert_slice: null argument");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_hubert_slice(static_cast<const __half*>(hidden), G, Tc, T, D, B, R, start, mult, win_l, out_f32,
                                      static_cast<__half*>(out_nhwc), c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("hubert_slice: ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_vae_post(ltb_ctx* c, const void* x, long long npix, int Ctot, void* out_u8) {
  if (!c || !x || !out_u8) return LTB_FAIL("vae_post: null argument");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_vae_post(static_cast<const __half*>(x), (size_t)npix, Ctot, static_cast<uint8_t*>(out_u8), c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("vae_post: ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_bgr_to_i420(ltb_ctx* c, const void* bgr_u8, int N, int H, int W, void* out_i420) {
  if (!c || !bgr_u8 || !out_i420) return LTB_FAIL("bgr_to_i420: null argument");
  LTB_CTX_ENTER(c);
  if (N <= 0 || H <= 0 || W <= 0 || (H & 1) || (W & 3)) return LTB_FAIL("bgr_to_i420: needs even height and a width that is a multiple of 4");
  cudaError_t e = launch_bgr_to_i420(static_cast<const uint8_t*>(bgr_u8), N, H, W, static_cast<uint8_t*>(out_i420), c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("bgr_to_i420: ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_stamp_pixels(ltb_ctx* c, void* frames_u8, int N, int H, int W, const void* pix_yx, int n, int b, int g, int r) {
  if (!c || !frames_u8 || (!pix_yx && n > 0)) return LTB_FAIL("stamp_pixels: null argument");
  if (N < 0 || n < 0 || H <= 0 || W <= 0) return LTB_FAIL("stamp_pixels: bad size");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_stamp_pixels(static_cast<uint8_t*>(frames_u8), N, H, W, static_cast<const int*>(pix_yx), n, b, g, r, c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("stamp_pixels: ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
// ---- S3FD face detector glue (s3fd.cu)
int ltb_op_s3fd_prep(ltb_ctx* c, const void* bgr_u8, int N, int H, int W, void* out) {
  if (!c || !bgr_u8 || !out) return LTB_FAIL("s3fd_prep: null argument");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_s3fd_prep(static_cast<const uint8_t*>(bgr_u8), N, H, W, static_cast<__half*>(out), c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("s3fd_prep (N, H, W > 0, 16-byte aligned output): ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_maxpool2x2(ltb_ctx* c, const void* x, int N, int H, int W, int C, void* out) {
  if (!c || !x || !out) return LTB_FAIL("maxpool2x2: null argument");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_maxpool2x2(static_cast<const __half*>(x), N, H, W, C, static_cast<__half*>(out), c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("maxpool2x2 (H, W >= 2, C % 8 == 0, 16-byte aligned): ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_l2norm(ltb_ctx* c, const void* x, long long npix, int C, const float* w, float eps, void* out) {
  if (!c || !x || !w || !out) return LTB_FAIL("l2norm: null argument");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_l2norm_scale(static_cast<const __half*>(x), npix, C, w, eps, static_cast<__half*>(out), c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("l2norm (C % 8 == 0, C <= 512, 16-byte aligned): ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_s3fd_select(ltb_ctx* c, const void* const* heads6, const int* hw12, int N, int pitch, float thresh, int* out_i32, float* out_score) {
  if (!c || !heads6 || !hw12 || !out_i32 || !out_score) return LTB_FAIL("s3fd_select: null argument");
  if (pitch < 8 || (pitch & 7)) return LTB_FAIL("s3fd_select: the head pitch must be a multiple of 8");
  LTB_CTX_ENTER(c);
  S3fdHeads h;
  for (int l = 0; l < kS3fdLevels; ++l) {
    h.p[l] = static_cast<const __half*>(heads6[l]);
    h.h[l] = hw12[2 * l];
    h.w[l] = hw12[2 * l + 1];
  }
  h.pitch = pitch;
  cudaError_t e = launch_s3fd_select(h, N, thresh, out_i32, out_score, c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("s3fd_select: ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
// ---- PFLD landmark network glue (pfld.cu)
int ltb_op_pfld_prep(ltb_ctx* c, const void* bgr_u8, int N, int H, int W, void* out) {
  if (!c || !bgr_u8 || !out) return LTB_FAIL("pfld_prep: null argument");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_pfld_prep(static_cast<const uint8_t*>(bgr_u8), N, H, W, static_cast<__half*>(out), c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("pfld_prep (N, H, W > 0, 16-byte aligned output): ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_pfld_head(ltb_ctx* c, const void* const* taps5, const int* hw5, const int* pitch5, const int* nch5, const int* ch, int N,
                     const float* wt, const float* bias, const float* mean, const int* crop_wh, int nout, float* out_f32, int* out_i32) {
  if (!c || !taps5 || !hw5 || !pitch5 || !nch5 || !ch || !wt || !bias || !mean || !crop_wh || !out_f32 || !out_i32)
    return LTB_FAIL("pfld_head: null argument");
  PfldTaps t{};
  int nfeat = 0;
  for (int k = 0; k < kPfldTaps; ++k) {
    t.p[k] = static_cast<const __half*>(taps5[k]);
    t.hw[k] = hw5[k];
    t.pitch[k] = pitch5[k];
    t.nch[k] = nch5[k];
    if (nch5[k] < 0 || nch5[k] > kPfldMaxFeat - nfeat) return LTB_FAIL("pfld_head: more than 256 features");
    nfeat += nch5[k];
  }
  for (int j = 0; j < nfeat; ++j) {
    if (ch[j] < 0 || ch[j] >= kPfldMaxPitch) return LTB_FAIL("pfld_head: channel index outside the pitch");
    t.ch[j] = (unsigned char)ch[j];
  }
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_pfld_head(t, N, wt, bias, mean, crop_wh, nout, out_f32, out_i32, c->st);
  if (e != cudaSuccess)
    return LTB_FAIL(std::string("pfld_head (pitch % 8 == 0 and <= 256, channels inside the pitch, 16-byte aligned taps, even nout <= 512): ") +
                    cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
// ---- BiSeNet face-parsing glue (bisenet.cu)
int ltb_op_bisenet_prep(ltb_ctx* c, const void* rgb_u8, int N, void* out) {
  if (!c || !rgb_u8 || !out) return LTB_FAIL("bisenet_prep: null argument");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_bisenet_prep(static_cast<const uint8_t*>(rgb_u8), N, static_cast<__half*>(out), c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("bisenet_prep (N > 0, 16-byte aligned output): ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_maxpool3x3s2(ltb_ctx* c, const void* x, int N, int H, int W, int C, void* out) {
  if (!c || !x || !out) return LTB_FAIL("maxpool3x3s2: null argument");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_maxpool3x3s2(static_cast<const __half*>(x), N, H, W, C, static_cast<__half*>(out), c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("maxpool3x3s2 (C % 8 == 0, 16-byte aligned): ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_chan_gate(ltb_ctx* c, const void* x, int N, int HW, int C, int pitch, int c_off, const float* w1t, const float* b1, int n1, int act1,
                     const float* w2t, const float* b2, int n2, int act2, float* out) {
  if (!c || !x || !w1t || !out) return LTB_FAIL("chan_gate: null argument");
  ChanGateArgs a{static_cast<const __half*>(x), N, HW, C, pitch, c_off, w1t, b1, n1, act1, w2t, b2, n2, act2, out};
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_chan_gate(a, c->st);
  if (e != cudaSuccess)
    return LTB_FAIL(std::string("chan_gate (C, pitch, c_off % 8 == 0, C, n1, n2 <= 512, act in 0..2, 16-byte aligned x): ") +
                    cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_chan_scale_add(ltb_ctx* c, const void* x, int N, int HW, int C, int xpitch, int xoff, const float* g, int mode, const float* yvec,
                          const void* y, int ypitch, int yoff, void* out, int opitch, int ooff) {
  if (!c || !x || !g || !out) return LTB_FAIL("chan_scale_add: null argument");
  ChanScaleAddArgs a{static_cast<const __half*>(x), N, HW, C, xpitch, xoff, g, mode, yvec, static_cast<const __half*>(y), ypitch, yoff,
                     static_cast<__half*>(out), opitch, ooff};
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_chan_scale_add(a, c->st);
  if (e != cudaSuccess)
    return LTB_FAIL(std::string("chan_scale_add (C, pitches, offsets % 8 == 0, mode 0..2 with its operand, 16-byte aligned): ") +
                    cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_bisenet_upsample_argmax(ltb_ctx* c, const void* logits, int N, int IH, int IW, int pitch, int ncls, int OH, int OW, void* labels) {
  if (!c || !logits || !labels) return LTB_FAIL("bisenet_upsample_argmax: null argument");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_bisenet_upsample_argmax(static_cast<const __half*>(logits), N, IH, IW, pitch, ncls, OH, OW, static_cast<uint8_t*>(labels),
                                                 c->st);
  if (e != cudaSuccess)
    return LTB_FAIL(std::string("bisenet_upsample_argmax (pitch % 8 == 0 covering ncls rounded up to 8, 16-byte aligned logits): ") +
                    cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_vae_pre(ltb_ctx* c, const void* img_u8, int N, int H, int W, int half_mask, void* out) {
  if (!c || !img_u8 || !out) return LTB_FAIL("vae_pre: null argument");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_vae_pre(static_cast<const uint8_t*>(img_u8), N, H, W, half_mask, static_cast<__half*>(out), c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("vae_pre: ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_gather_rows(ltb_ctx* c, const void* table, int n, const void* d_index, int B, long long row_elems, void* out) {
  if (!c || !table || !d_index || !out) return LTB_FAIL("gather_rows: null argument");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_gather_rows(static_cast<const __half*>(table), n, static_cast<const int*>(d_index), B, (size_t)row_elems,
                                     static_cast<__half*>(out), c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("gather_rows: ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_whisper_logmel_grouped(ltb_ctx* c, const void* pcm_f32, int G, int n, const void* fb_f32, void* logspec_ws, void* gmax_ws,
                                  void* out_f16, void* out_f32) {
  if (!c || !pcm_f32 || !fb_f32 || !logspec_ws || !gmax_ws || !out_f16) return LTB_FAIL("whisper_logmel: null argument");
  LTB_CTX_ENTER(c);
  cudaError_t e = launch_whisper_logmel(static_cast<const float*>(pcm_f32), G, n, static_cast<const float*>(fb_f32),
                                        static_cast<float*>(logspec_ws), static_cast<int*>(gmax_ws), static_cast<__half*>(out_f16),
                                        static_cast<float*>(out_f32), c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("whisper_logmel (1 <= n <= 480000, 1 <= G <= 65535): ") + cudaGetErrorString(e));
  c->launches += 3;
  return 0;
}
int ltb_op_whisper_slice_grouped(ltb_ctx* c, const void* const* hidden5, int G, int T, int D, int B, float start, float mult, void* out,
                                 int out_rows_per_frame) {
  if (!c || !hidden5 || !out) return LTB_FAIL("whisper_slice: null argument");
  LTB_CTX_ENTER(c);
  if (D % 8 != 0 || out_rows_per_frame < 50) return LTB_FAIL("whisper_slice: bad shape");
  cudaError_t e = launch_whisper_slice(reinterpret_cast<const __half* const*>(hidden5), G, T, D, B, start, mult, static_cast<__half*>(out),
                                       out_rows_per_frame, c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("whisper_slice (T >= 1, 1 <= B, G <= 65535): ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}
int ltb_op_mt_paste(ltb_ctx* c, const ltb_mt_paste_op* d) {
  if (!c || !d) return LTB_FAIL("mt_paste: null argument");
  LTB_CTX_ENTER(c);
  MtPasteArgs a;
  a.frames = static_cast<const uint8_t*>(d->frames);
  a.coords = static_cast<const int*>(d->coords);
  a.crop = static_cast<const int*>(d->crop);
  a.masks = static_cast<const uint8_t*>(d->masks);
  a.mask_off = static_cast<const long long*>(d->mask_off);
  a.pred = static_cast<const uint8_t*>(d->pred);
  a.out = static_cast<uint8_t*>(d->out);
  a.nf = d->nf;
  a.H = d->H;
  a.W = d->W;
  a.index = d->index;
  a.explicit_idx = d->explicit_idx;
  a.slot0 = d->slot0;
  a.S = d->pred_hw > 0 ? d->pred_hw : 256;
  cudaError_t e = launch_mt_paste(a, d->count, c->st);
  if (e != cudaSuccess) return LTB_FAIL(std::string("mt_paste: ") + cudaGetErrorString(e));
  c->launches += 1;
  return 0;
}

}  // extern "C"
