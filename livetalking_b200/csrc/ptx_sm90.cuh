// Thin inline-PTX wrappers for the sm_90a features the engine uses:
// mbarrier, cp.async, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA), proxy fences.
// sm_90a only — there is no fallback path.
#pragma once
#include <cuda_fp16.h>
#include <cstdint>
#include <cstdio>

namespace ltb {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a pipeline bug turns into a trap (reported as a CUDA error by the host API) instead of a hung GPU.
// ~4 s at 2 GHz.  No function call in here: a call between wgmma issues makes ptxas serialise the wgmma pipeline.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 8000000000LL) __trap();
  }
}

// ---------------------------------------------------------------- fences
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---------------------------------------------------------------- cp.async (LDGSTS)
// 16-byte copy; src_bytes = 0 zero-fills the destination (used for conv padding / tile tails).
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
  return v;
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
      "l"(tmap), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(dst),
      "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(
          dst),
      "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, int c2, int c3,
                                            int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::
          "r"(dst),
      "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}

// ---------------------------------------------------------------- ldmatrix
// four 8x8 b16 matrices; lanes 8k..8k+7 give the 16-byte row addresses of matrix k, and lane l receives row l/4, elements
// 2(l%4) (+1) of each matrix: the wgmma accumulator fragment layout of one 8-row x 8-column block
__device__ __forceinline__ void ldmatrix_x4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, uint32_t saddr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(saddr)
               : "memory");
}

// the same four matrices transposed: lane l receives column l/4, elements 2(l%4) (+1), i.e. (row 2(l%4) (+1), column l/4)
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, uint32_t saddr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(saddr)
               : "memory");
}
// inverse of ldmatrix_x4_trans: lane l's words are (row 2(l%4) (+1), column l/4) of the four matrices whose row addresses
// lanes 8k..8k+7 give
__device__ __forceinline__ void stmatrix_x4_trans(uint32_t saddr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.trans.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(saddr), "r"(r0), "r"(r1), "r"(r2), "r"(r3)
               : "memory");
}

// ---------------------------------------------------------------- TMA store (bulk async group)
__device__ __forceinline__ void tma_store_4d(const void* tmap, uint32_t src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(tmap), "r"(src), "r"(c0),
               "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// the shared-memory sources of all but the newest N bulk groups have been read (they may be overwritten)
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
// the bulk groups but the newest N have completed their global writes
template <int N>
__device__ __forceinline__ void bulk_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ---------------------------------------------------------------- named barriers (id 0 is __syncthreads)
__device__ __forceinline__ void named_sync(uint32_t id, uint32_t threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
__device__ __forceinline__ void named_arrive(uint32_t id, uint32_t threads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// ---------------------------------------------------------------- wgmma (sm_90a warpgroup MMA)
// K-major shared-memory matrix descriptor: rows of the swizzle span (128 / 64 / 32 B) packed densely, 8-row core groups SBO
// bytes apart; LBO is the distance between K-adjacent core matrices (used by SWIZZLE_NONE only).
//   layout: 0 = SWIZZLE_NONE, 1 = SWIZZLE_128B, 2 = SWIZZLE_64B, 3 = SWIZZLE_32B
// The swizzle is applied to the absolute shared-memory address, so a start address that is not a multiple of the 1024-byte
// pattern (a shifted im2col view into a halo tile) reads the rows TMA wrote there.
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t layout) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)(layout & 3) << 62;
  return d;
}
// high word of a SWIZZLE_128B K-major descriptor with the given SBO; the low word is (addr >> 4) | (1 << 16) (LBO = 16 B)
__host__ __device__ constexpr uint32_t wgmma_hi_128b(uint32_t sbo_bytes) { return (sbo_bytes >> 4) | (1u << 30); }
// the same for SWIZZLE_32B (32-byte rows: one k16 step of fp16 per row)
__host__ __device__ constexpr uint32_t wgmma_hi_32b(uint32_t sbo_bytes) { return (sbo_bytes >> 4) | (3u << 30); }
__device__ __forceinline__ uint32_t wgmma_lo(uint32_t saddr) { return ((saddr & 0x3FFFFu) >> 4) | (1u << 16); }
__device__ __forceinline__ uint64_t wgmma_lohi(uint32_t lo, uint32_t hi) { return ((uint64_t)hi << 32) | lo; }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across an in-flight wgmma
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D (64 x N fp32, registers of the issuing warpgroup) (+)= A (64 x 16) * B (N x 16)^T, fp16 in.
//   ss: A and B from shared-memory descriptors; rs: A from registers (the m64k16 fp16 fragment layout).
//   Only the shapes the kernels use are instantiated.
// Accumulator layout: warp w of the warpgroup, lane l holds rows 16w + l/4 (+8) and columns 8i + 2(l%4) (+1):
//   d[4i + 0..1] -> row 16w + l/4, d[4i + 2..3] -> row 16w + l/4 + 8.
template <int N>
struct Wgmma;
// accumulator operand lists: LTB_D<n>(i) = "+f"(d[i]), ..., "+f"(d[i + n - 1])
#define LTB_D1(i) "+f"(d[i])
#define LTB_D2(i) LTB_D1(i), LTB_D1(i + 1)
#define LTB_D4(i) LTB_D2(i), LTB_D2(i + 2)
#define LTB_D8(i) LTB_D4(i), LTB_D4(i + 4)
#define LTB_D16(i) LTB_D8(i), LTB_D8(i + 8)
#define LTB_D32(i) LTB_D16(i), LTB_D16(i + 16)
#define LTB_D64(i) LTB_D32(i), LTB_D32(i + 32)
#define LTB_D128(i) LTB_D64(i), LTB_D64(i + 64)
#define LTB_WG_HEAD(P) "{\n.reg .pred p;\nsetp.ne.b32 p, %" P ", 0;\nwgmma.mma_async.sync.aligned.m64n"
#define LTB_WG_SS(N, REGS, A, B, P) LTB_WG_HEAD(P) N "k16.f32.f16.f16 " REGS ", %" A ", %" B ", p, 1, 1, 0, 0;\n}\n"
#define LTB_WG_RS(N, REGS, A, B, P) \
  LTB_WG_HEAD(P) N "k16.f32.f16.f16 " REGS ", {%" A "}, %" B ", p, 1, 1, 0;\n}\n"

template <>
struct Wgmma<16> {
#define LTB_R "{%0,%1,%2,%3,%4,%5,%6,%7}"
  __device__ __forceinline__ static void ss(float (&d)[8], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(LTB_WG_SS("16", LTB_R, "8", "9", "10") : LTB_D8(0) : "l"(a), "l"(b), "r"(acc));
  }
  __device__ __forceinline__ static void rs(float (&d)[8], const uint32_t (&a)[4], uint64_t b, uint32_t acc) {
    asm volatile(LTB_WG_RS("16", LTB_R, "8,%9,%10,%11", "12", "13") : LTB_D8(0)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc));
  }
#undef LTB_R
};

template <>
struct Wgmma<32> {
#define LTB_R "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}"
  __device__ __forceinline__ static void ss(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(LTB_WG_SS("32", LTB_R, "16", "17", "18") : LTB_D16(0) : "l"(a), "l"(b), "r"(acc));
  }
  __device__ __forceinline__ static void rs(float (&d)[16], const uint32_t (&a)[4], uint64_t b, uint32_t acc) {
    asm volatile(LTB_WG_RS("32", LTB_R, "16,%17,%18,%19", "20", "21") : LTB_D16(0)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc));
  }
#undef LTB_R
};

template <>
struct Wgmma<48> {
#define LTB_R "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23}"
  __device__ __forceinline__ static void rs(float (&d)[24], const uint32_t (&a)[4], uint64_t b, uint32_t acc) {
    asm volatile(LTB_WG_RS("48", LTB_R, "24,%25,%26,%27", "28", "29") : LTB_D16(0), LTB_D8(16)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc));
  }
#undef LTB_R
};

template <>
struct Wgmma<64> {
#define LTB_R "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}"
  __device__ __forceinline__ static void ss(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(LTB_WG_SS("64", LTB_R, "32", "33", "34") : LTB_D32(0) : "l"(a), "l"(b), "r"(acc));
  }
  __device__ __forceinline__ static void rs(float (&d)[32], const uint32_t (&a)[4], uint64_t b, uint32_t acc) {
    asm volatile(LTB_WG_RS("64", LTB_R, "32,%33,%34,%35", "36", "37") : LTB_D32(0)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc));
  }
#undef LTB_R
};

template <>
struct Wgmma<80> {
#define LTB_R "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39}"
  __device__ __forceinline__ static void rs(float (&d)[40], const uint32_t (&a)[4], uint64_t b, uint32_t acc) {
    asm volatile(LTB_WG_RS("80", LTB_R, "40,%41,%42,%43", "44", "45") : LTB_D32(0), LTB_D8(32)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc));
  }
#undef LTB_R
};

template <>
struct Wgmma<96> {
#define LTB_R "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47}"
  __device__ __forceinline__ static void ss(float (&d)[48], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(LTB_WG_SS("96", LTB_R, "48", "49", "50") : LTB_D32(0), LTB_D16(32) : "l"(a), "l"(b), "r"(acc));
  }
  __device__ __forceinline__ static void rs(float (&d)[48], const uint32_t (&a)[4], uint64_t b, uint32_t acc) {
    asm volatile(LTB_WG_RS("96", LTB_R, "48,%49,%50,%51", "52", "53") : LTB_D32(0), LTB_D16(32)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc));
  }
#undef LTB_R
};

template <>
struct Wgmma<112> {
#define LTB_R "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55}"
  __device__ __forceinline__ static void rs(float (&d)[56], const uint32_t (&a)[4], uint64_t b, uint32_t acc) {
    asm volatile(LTB_WG_RS("112", LTB_R, "56,%57,%58,%59", "60", "61") : LTB_D32(0), LTB_D16(32), LTB_D8(48)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc));
  }
#undef LTB_R
};

template <>
struct Wgmma<128> {
#define LTB_R "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}"
  __device__ __forceinline__ static void ss(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(LTB_WG_SS("128", LTB_R, "64", "65", "66") : LTB_D64(0) : "l"(a), "l"(b), "r"(acc));
  }
  __device__ __forceinline__ static void rs(float (&d)[64], const uint32_t (&a)[4], uint64_t b, uint32_t acc) {
    asm volatile(LTB_WG_RS("128", LTB_R, "64,%65,%66,%67", "68", "69") : LTB_D64(0)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc));
  }
#undef LTB_R
};

template <>
struct Wgmma<144> {
#define LTB_R "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71}"
  __device__ __forceinline__ static void rs(float (&d)[72], const uint32_t (&a)[4], uint64_t b, uint32_t acc) {
    asm volatile(LTB_WG_RS("144", LTB_R, "72,%73,%74,%75", "76", "77") : LTB_D64(0), LTB_D8(64)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc));
  }
#undef LTB_R
};

template <>
struct Wgmma<160> {
#define LTB_R "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79}"
  __device__ __forceinline__ static void rs(float (&d)[80], const uint32_t (&a)[4], uint64_t b, uint32_t acc) {
    asm volatile(LTB_WG_RS("160", LTB_R, "80,%81,%82,%83", "84", "85") : LTB_D64(0), LTB_D16(64)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc));
  }
#undef LTB_R
};

template <>
struct Wgmma<192> {
#define LTB_R "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95}"
  __device__ __forceinline__ static void ss(float (&d)[96], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(LTB_WG_SS("192", LTB_R, "96", "97", "98") : LTB_D64(0), LTB_D32(64) : "l"(a), "l"(b), "r"(acc));
  }
#undef LTB_R
};

template <>
struct Wgmma<256> {
#define LTB_R "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}"
  __device__ __forceinline__ static void ss(float (&d)[128], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(LTB_WG_SS("256", LTB_R, "128", "129", "130") : LTB_D128(0) : "l"(a), "l"(b), "r"(acc));
  }
#undef LTB_R
};

// call Wgmma<N> on accumulator columns [c0, c0 + N) of a wider register tile (c0 a compile-time multiple of 8)
template <int N, int C0, int R>
__device__ __forceinline__ void wgmma_ss_at(float (&d)[R], uint64_t a, uint64_t b, uint32_t acc) {
  static_assert(C0 % 8 == 0 && C0 / 2 + N / 2 <= R, "accumulator slice out of range");
  Wgmma<N>::ss(*reinterpret_cast<float(*)[N / 2]>(&d[C0 / 2]), a, b, acc);
}

// fp32 pair -> packed fp16x2 with saturation to +-65504 (and ReLU) in ONE instruction (F2FP.SATFINITE[.RELU].F16.F32.PACK_AB):
// replaces convert + max(0) + min(65504) of the epilogue (3 instructions per channel pair).  Result: {lo, hi} = half2(lo, hi).
__device__ __forceinline__ uint32_t f32x2_to_f16x2_sat(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ uint32_t f32x2_to_f16x2_sat_relu(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.relu.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}

// Programmatic dependent launch: a kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may start
// while its predecessor in the stream is still running; everything that touches the predecessor's output (or overwrites
// its input) must come after pdl_wait(), which returns once the predecessor grid has completed and flushed.  Both are
// no-ops for a normal launch.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// Warpgroup register reallocation: every thread of the warpgroup executes it; the kernel's register count (from
// __launch_bounds__) must be the per-thread budget the warpgroups trade within.
template <uint32_t N>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}
template <uint32_t N>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}

// ---------------------------------------------------------------- thread-block clusters (distributed shared memory)
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// every thread of every CTA of the cluster arrives; shared-memory writes before it are visible to the cluster after it
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// the address of the same shared-memory location in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t dsmem_map(uint32_t saddr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(saddr), "r"(rank));
  return r;
}
__device__ __forceinline__ float4 dsmem_ld_f32x4(uint32_t caddr) {
  float4 v;
  asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(caddr) : "memory");
  return v;
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

}  // namespace ltb
