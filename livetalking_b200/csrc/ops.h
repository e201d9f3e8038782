// Launchers of the bandwidth-bound operators (ops.cu) and the MuseTalk blend composite (mt_paste.cu).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cstddef>
#include <cstdint>

namespace ltb {

cudaError_t launch_groupnorm(const __half* x, int N, int HW, int C, int Ctot, int c_off, int groups, float eps, const float* gamma,
                             const float* beta, int silu, __half* out, int OCtot, int oc_off, float* stats_ws, cudaStream_t st);
cudaError_t launch_gn_stats(const __half* x, int N, int HW, int C, int Ctot, int c_off, int groups, float* stats, cudaStream_t st);
cudaError_t launch_gn_apply(const __half* x, int N, int HW, int C, int Ctot, int c_off, int groups, float eps, const float* stats,
                            const float* gamma, const float* beta, int silu, __half* out, int OCtot, int oc_off, cudaStream_t st);
cudaError_t launch_layernorm(const __half* x, int rows, int C, float eps, const float* gamma, const float* beta, __half* out,
                             cudaStream_t st);
cudaError_t launch_softmax(const __half* x, int rows, int cols, int ld, int valid, float scale, __half* out, cudaStream_t st);
cudaError_t launch_geglu(const __half* h, size_t rows, int H, __half* out, cudaStream_t st);
cudaError_t launch_eltwise(const __half* x, const __half* y, size_t n, size_t period, int act, __half* out, cudaStream_t st);
cudaError_t launch_upsample2x(const __half* x, int N, int H, int W, int C, __half* out, cudaStream_t st);
cudaError_t launch_copy_channels(const __half* src, size_t rows, int C, int SCtot, int sc_off, __half* dst, int DCtot, int dc_off,
                                 cudaStream_t st);
cudaError_t launch_transpose_heads(const __half* v, int B, int n_keys, int Ctot, int c_off, int heads, int d, int n_pad, __half* vt,
                                   cudaStream_t st);
// softmax(scale * Q K^T) V in one kernel (attn_fused.cu); head dim d % 16 == 0, d <= 160
bool attn_fused_supported(int d, int q_pitch, int kv_pitch, int n_pad);
cudaError_t launch_attn_fused(const __half* q, int q_pitch, const __half* k, int kv_pitch, int kv_rows, const __half* vt, int n_pad, int B, int H,
                              int nq, int valid, int d, float scale, __half* out, int out_pitch, cudaStream_t st);
// ---- UltraLight / HuBERT (ultralight.cu, hubert.cu)
// grouped weights of the per-image ops: image n uses w + s * w_stride and bias + s * b_stride, s = slot[n / images] (device table)
struct WeightGroups {
  const int* slot;
  int images;
  long long w_stride, b_stride;
};
// grp == nullptr: ungrouped
cudaError_t launch_dwconv3x3(const __half* x, int N, int IH, int IW, int ICtot, int ic_off, int C, const __half* w, const float* bias, int stride,
                             int relu, __half* out, int OCtot, int oc_off, cudaStream_t st, const WeightGroups* grp = nullptr);
// per-group crop source of launch_ul_prep_grouped (layout of ltb_ul_prep_group)
struct UlPrepGroup {
  const uint8_t* faces;
  int nf, index;
};
cudaError_t launch_ul_prep_grouped(const UlPrepGroup* groups, int group_images, int B, __half* out, cudaStream_t st);
// 32 -> 3 head + sigmoid * 255 (w2l_small.cu); grouped: hw pixels per image, hw % 256 == 0
cudaError_t launch_head_grouped(const __half* x, const float* w3x32, const float* b3, float* pred, int npix, int hw, const WeightGroups& grp,
                                cudaStream_t st);
cudaError_t launch_upsample_bilinear2x(const __half* x, int N, int H, int W, int ICtot, int ic_off, int C, __half* out, int OCtot, int oc_off,
                                       cudaStream_t st);
cudaError_t launch_ul_prep(const uint8_t* faces, int nf, const int* d_index, int B, __half* out, cudaStream_t st);
cudaError_t launch_ul_paste(const uint8_t* frames, const uint8_t* faces, const int* coords, const float* pred, uint8_t* out, int nf, int H, int W,
                            int index, int explicit_idx, int slot0, int count, cudaStream_t st);
// HuBERT ops over G sequences stacked on the row dimension (G = 1: one window)
cudaError_t launch_hubert_conv0(const float* pcm, int G, int n, const float* w, const float* bias, int C, float* stats, __half* out,
                                cudaStream_t st);
cudaError_t launch_hubert_pos_conv(const __half* h, int G, int T, int D, int groups, int K, const __half* w, const float* bias, __half* out,
                                   cudaStream_t st);
cudaError_t launch_hubert_slice(const __half* hidden, int G, int Tc, int T, int D, int B, int R, float start, float mult, int win_l,
                                float* out_f32, __half* out_nhwc, cudaStream_t st);
cudaError_t launch_vae_post(const __half* x, size_t npix, int Ctot, uint8_t* out, cudaStream_t st);
// uint8 BGR [N,H,W,3] -> planar I420 [N, H*3/2, W] (OpenCV COLOR_BGR2YUV_I420 arithmetic); H even, W % 4 == 0
cudaError_t launch_bgr_to_i420(const uint8_t* bgr, int N, int H, int W, uint8_t* out, cudaStream_t st);
cudaError_t launch_stamp_pixels(uint8_t* frames, int N, int H, int W, const int* pix, int n, int b, int g, int r, cudaStream_t st);
cudaError_t launch_vae_pre(const uint8_t* img, int N, int H, int W, int half_mask, __half* out, cudaStream_t st);
cudaError_t launch_gather_rows(const __half* table, int n, const int* d_index, int B, size_t row_elems, __half* out, cudaStream_t st);

// Whisper front-end (whisper.cu)
cudaError_t launch_whisper_logmel(const float* pcm, int n, const float* fb, float* logspec_ws, int* gmax, __half* out16, float* out32,
                                  cudaStream_t st);
cudaError_t launch_whisper_slice(const __half* const* hidden5, int T, int D, int B, float start, float mult, __half* out,
                                 int out_rows_per_frame, cudaStream_t st);

// MuseTalk paste-back (mt_paste.cu): resize + insert + blendLinear, `count` frames per launch
struct MtPasteArgs {
  const uint8_t* frames;     // [nf,H,W,3]
  const int* coords;         // [nf,4] = (x1,y1,x2,y2)           (musetalk_avatar.py:157)
  const int* crop;           // [nf,4] = (x_s,y_s,x_e,y_e)       (myutil.py:7)
  const uint8_t* masks;      // concatenated 3-channel masks, frame i at mask_off[i], size (y_e-y_s) x (x_e-x_s) x 3
  const long long* mask_off;
  const uint8_t* pred;       // [B,S,S,3] u8 BGR (VAE decode output)
  uint8_t* out;              // [count,H,W,3]
  int nf, H, W;
  int index, explicit_idx, slot0;
  int S;                     // prediction side: 256 (reference), 512 for the 64x64-latent configuration
};
cudaError_t launch_mt_paste(const MtPasteArgs& a, int count, cudaStream_t st);

// S3FD face detector glue (s3fd.cu)
constexpr int kS3fdInC = 16;     // channels of the prepared image: RGB minus means, zero-padded (conv1_1 runs with Cin = 16)
constexpr int kS3fdLevels = 6;
struct S3fdHeads {               // the six fused conf + loc head outputs, [N][h][w][pitch] fp16 each
  const __half* p[kS3fdLevels];
  int h[kS3fdLevels], w[kS3fdLevels];
  int pitch;
};
cudaError_t launch_s3fd_prep(const uint8_t* bgr, int N, int H, int W, __half* out, cudaStream_t st);
cudaError_t launch_maxpool2x2(const __half* x, int N, int H, int W, int C, __half* out, cudaStream_t st);
cudaError_t launch_l2norm_scale(const __half* x, long long npix, int C, const float* w, float eps, __half* out, cudaStream_t st);
cudaError_t launch_s3fd_select(const S3fdHeads& heads, int N, float thresh, int* out_i, float* out_s, cudaStream_t st);

// PFLD landmark network glue (pfld.cu)
constexpr int kPfldInC = 16;       // channels of the prepared crop: BGR / 255, zero-padded (conv1 runs with Cin = 16)
constexpr int kPfldTaps = 5;       // x1..x4 (global average pools) and x5 (conv8, 1 x 1)
constexpr int kPfldMaxPitch = 256;
constexpr int kPfldMaxFeat = 256;
struct PfldTaps {                  // tap t: [N][hw[t]][pitch[t]] fp16; its nch[t] real channels are listed in ch, taps in order
  const __half* p[kPfldTaps];
  int hw[kPfldTaps], pitch[kPfldTaps], nch[kPfldTaps];
  unsigned char ch[kPfldMaxFeat];
};
cudaError_t launch_pfld_prep(const uint8_t* bgr, int N, int H, int W, __half* out, cudaStream_t st);
cudaError_t launch_pfld_head(const PfldTaps& taps, int N, const float* wt, const float* bias, const float* mean, const int* crop_wh, int nout,
                             float* out_f, int* out_i, cudaStream_t st);

// BiSeNet face-parsing glue (bisenet.cu)
constexpr int kBisenetIn = 512;    // FaceParsing resizes every crop to 512 x 512
constexpr int kBisenetS2d = 259;   // space-to-depth 2 x 2 map of the stem: 2 pixels of zero border before, 1 after
constexpr int kBisenetInC = 16;    // 12 real channels ((by, bx, c) order), zero-padded
constexpr int kChanGateMax = 512;  // chan_gate: largest C, n1, n2
enum { kActNone = 0, kActRelu = 1, kActSigmoid = 2 };
enum { kScaleAddVec = 0, kScaleAddTensor = 1, kScaleAddSelf = 2 };
struct ChanGateArgs {              // x: [N][HW][pitch] fp16, channels [c_off, c_off + C); w1t fp32 [C][n1], w2t [n1][n2] (null: one layer)
  const __half* x;
  int N, HW, C, pitch, c_off;
  const float *w1t, *b1;
  int n1, act1;
  const float *w2t, *b2;
  int n2, act2;
  float* out;                      // [N][n2] (or [N][n1])
};
struct ChanScaleAddArgs {          // out = x * g[n][c] + (yvec[n][c] | y | x); x / y / out: [N][HW][pitch] fp16 channel slices
  const __half* x;
  int N, HW, C, xpitch, xoff;
  const float* g;
  int mode;
  const float* yvec;
  const __half* y;
  int ypitch, yoff;
  __half* out;
  int opitch, ooff;
};
cudaError_t launch_bisenet_prep(const uint8_t* rgb, int N, __half* out, cudaStream_t st);
cudaError_t launch_maxpool3x3s2(const __half* x, int N, int H, int W, int C, __half* out, cudaStream_t st);
cudaError_t launch_chan_gate(const ChanGateArgs& a, cudaStream_t st);
cudaError_t launch_chan_scale_add(const ChanScaleAddArgs& a, cudaStream_t st);
cudaError_t launch_bisenet_upsample_argmax(const __half* logits, int N, int IH, int IW, int pitch, int ncls, int OH, int OW, uint8_t* out,
                                           cudaStream_t st);

}  // namespace ltb
