// sm_90a primitives used by the tensor-core kernels: mbarrier, TMA (cp.async.bulk.tensor) and
// wgmma (warpgroup MMA: operands in shared memory, FP32 accumulators in registers) with its
// shared-memory matrix descriptors.  Inline PTX only.
//
// The pipeline the four GEMM kernels (conv16.cu, wgrad16.cu, conv_tc.cu, conv_tc_wgrad.cu)
// share: producers fill the slots of a shared-memory Ring (TMA, or gather + convert + store
// followed by fence_proxy_async) and complete the slot's full mbarrier; two consumer
// warpgroups of 64 tile rows each wait on it, issue the slot's wgmma as one commit group
// and release the slot on its empty mbarrier (one arrive per consumer warp) once the group
// has completed.  Ring::consume keeps one k-block of wgmma in flight while the next one is
// issued.  Split operands are multiplied by the three passes of mma3_*.  Epilogues work
// from the accumulator fragment: conv16 stages it per consumer warp in a shared-memory box
// that a TMA store (or reduce-add) writes out in the background, the other kernels store it
// straight to global memory; the conv epilogues sum BatchNorm statistics with
// stats_add / stats_flush in a fixed order.  Every mbarrier wait is bounded (trap instead of
// hang).
//
// wgmma shared-memory descriptor (PTX ISA "Matrix Descriptor Format"):
//   [0,14) start addr >> 4 | [16,30) leading byte offset >> 4 | [32,46) stride byte offset >> 4 |
//   [49,52) base offset (0: every tile is 1024-byte aligned) | [62,64) layout (1 = SWIZZLE_128B)
//
// Accumulator fragment of wgmma m64nN with FP32 D: thread t of the warpgroup holds, for
// j < N / 8 and h, e in {0, 1},
//   d[4j + 2h + e] = D[16 * (t / 32) + (t % 32) / 4 + 8h][8j + 2 * (t % 4) + e].
#pragma once
#include <cuda.h>
#include "common.cuh"

namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}

// ------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
// Bounded wait: a protocol bug traps (launch failure) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  long long t0 = 0;
  while (true) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity), "r"(2000u)
        : "memory");
    if (done) break;
    const long long now = clock64();            // the clock is read only when the wait blocks
    if (t0 == 0) t0 = now;
    if (now - t0 > 4000000000LL) __trap();      // ~2 s: protocol bug, fail loudly
  }
}

// generic-proxy smem writes -> visible to the async proxy (wgmma / TMA reads)
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// named barrier over `threads` threads (ids 1..15; 0 is __syncthreads)
__device__ __forceinline__ void named_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// ------------------------------------------------------------------ TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(m) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* m, uint32_t bar,
                                            int x, int y) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(dst), "l"(m), "r"(bar), "r"(x), "r"(y)
      : "memory");
}
// 3-D / 5-D loads (weight planes / activation planes of the split-fp16 path)
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* m, uint32_t bar,
                                            int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(dst), "l"(m), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap* m, uint32_t bar,
                                            int c0, int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::"r"(dst), "l"(m), "r"(bar), "r"(c0), "r"(c1),
      "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}

// TMA stores of an fp32 output box from (128B-swizzled) shared memory; bulk async-group completion
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, uint32_t src, int c0, int c1,
                                             int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(m),
      "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// out += box (element-wise fp32 add performed at L2)
__device__ __forceinline__ void tma_reduce_add_4d(const CUtensorMap* m, uint32_t src, int c0,
                                                  int c1, int c2, int c3) {
  asm volatile(
      "cp.reduce.async.bulk.tensor.4d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(m),
      "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_store_commit() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
// all but the newest N groups of this thread have finished READING their shared-memory source
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* m, uint32_t bar,
                                            int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(dst), "l"(m), "r"(bar), "r"(c0), "r"(c1),
      "r"(c2), "r"(c3)
      : "memory");
}

// ------------------------------------------------------------------ wgmma
__device__ __forceinline__ void wgmma_fence() {
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wgmma_commit() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
// all but the newest N committed groups of this warpgroup have completed
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator accesses across a wgmma fence / wait
template <int R>
__device__ __forceinline__ void fence_acc(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// K-major operand tile, 128-byte rows (64 fp16 / 32 tf32 of K), SWIZZLE_128B: 8-row atoms of
// 1024 B, stride between atoms (SBO) 1024 B; LBO is unused for swizzled K-major layouts
// (encoded 1).  `addr` lies in a 1024-byte aligned tile; the K step inside the 128-byte row
// is a plain byte offset on the start address.
__device__ __forceinline__ uint64_t desc_kmajor_sw128(uint32_t addr) {
  return (uint64_t)((addr & 0x3FFFF) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) |
         ((uint64_t)1 << 62);
}
// MN-major 16-bit operand, SWIZZLE_128B: 128-byte rows hold 64 consecutive MN elements of
// one k; 8 k-rows form a 1024 B atom (SBO = stride between k-atoms); LBO = byte stride
// between successive 64-element MN chunks (cute: ((8,8,m),(8,k)):((1,8,LBO),(64,SBO)) in
// fp16 elements).
__device__ __forceinline__ uint64_t desc_mnmajor16_sw128(uint32_t addr, uint32_t lbo_bytes,
                                                         uint32_t sbo_bytes) {
  return (uint64_t)((addr & 0x3FFFF) >> 4) | ((uint64_t)(lbo_bytes >> 4) << 16) |
         ((uint64_t)(sbo_bytes >> 4) << 32) | ((uint64_t)1 << 62);
}

// D (+)= A * B for one warpgroup, M = 64, N = 2 * (length of d); scale_d = 0 overwrites D.
#define EPB_ACC8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), \
                    "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
// f16: TA / TB = 1 for MN-major operands.  tf32: K-major operands only.
template <int TA, int TB>
__device__ __forceinline__ void wgmma_f16_n64(float (&d)[32], uint64_t adesc, uint64_t bdesc,
                                                int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17,"
      "%18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31},"
      " %32, %33, p, 1, 1, %35, %36;\n\t}"
      : EPB_ACC8(0), EPB_ACC8(8), EPB_ACC8(16), EPB_ACC8(24)
      : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_f16_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc,
                                                int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17,"
      "%18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34,"
      "%35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51,"
      "%52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63},"
      " %64, %65, p, 1, 1, %67, %68;\n\t}"
      : EPB_ACC8(0), EPB_ACC8(8), EPB_ACC8(16), EPB_ACC8(24), EPB_ACC8(32), EPB_ACC8(40), EPB_ACC8(48), EPB_ACC8(56)
      : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(TA), "n"(TB));
}

__device__ __forceinline__ void wgmma_tf32_n32(float (&d)[16], uint64_t adesc, uint64_t bdesc,
                                                 int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15},"
      " %16, %17, p, 1, 1;\n\t}"
      : EPB_ACC8(0), EPB_ACC8(8)
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}

__device__ __forceinline__ void wgmma_tf32_n64(float (&d)[32], uint64_t adesc, uint64_t bdesc,
                                                 int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17,"
      "%18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31},"
      " %32, %33, p, 1, 1;\n\t}"
      : EPB_ACC8(0), EPB_ACC8(8), EPB_ACC8(16), EPB_ACC8(24)
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}

__device__ __forceinline__ void wgmma_tf32_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc,
                                                 int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17,"
      "%18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34,"
      "%35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51,"
      "%52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63},"
      " %64, %65, p, 1, 1;\n\t}"
      : EPB_ACC8(0), EPB_ACC8(8), EPB_ACC8(16), EPB_ACC8(24), EPB_ACC8(32), EPB_ACC8(40), EPB_ACC8(48), EPB_ACC8(56)
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_f16(float (&d)[32], uint64_t a, uint64_t b, int sd) {
  wgmma_f16_n64<TA, TB>(d, a, b, sd);
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_f16(float (&d)[64], uint64_t a, uint64_t b, int sd) {
  wgmma_f16_n128<TA, TB>(d, a, b, sd);
}
__device__ __forceinline__ void wgmma_tf32(float (&d)[16], uint64_t a, uint64_t b, int sd) {
  wgmma_tf32_n32(d, a, b, sd);
}
__device__ __forceinline__ void wgmma_tf32(float (&d)[32], uint64_t a, uint64_t b, int sd) {
  wgmma_tf32_n64(d, a, b, sd);
}
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], uint64_t a, uint64_t b, int sd) {
  wgmma_tf32_n128(d, a, b, sd);
}

// Error-compensated products of one k-step: a*b ~= a_lo*b_hi + a_hi*b_lo + a_hi*b_hi.  The
// passes are issued in this order; outputs are bit-identical run to run and build to build
// only while it stays the same.
template <int TA, int TB, int R>
__device__ __forceinline__ void mma3_f16(float (&d)[R], uint64_t ah, uint64_t al, uint64_t bh,
                                         uint64_t bl) {
  wgmma_f16<TA, TB>(d, al, bh, 1);
  wgmma_f16<TA, TB>(d, ah, bl, 1);
  wgmma_f16<TA, TB>(d, ah, bh, 1);
}
template <int R>
__device__ __forceinline__ void mma3_tf32(float (&d)[R], uint64_t ah, uint64_t al, uint64_t bh,
                                          uint64_t bl) {
  wgmma_tf32(d, al, bh, 1);
  wgmma_tf32(d, ah, bl, 1);
  wgmma_tf32(d, ah, bh, 1);
}

// ------------------------------------------------------------------ operand ring
// S operand slots of STAGE bytes with a full and an empty mbarrier per slot (8 bytes apart
// from full(0) / empty(0)).  Offsets count from the 1024-byte aligned start `sm` of dynamic
// shared memory (SWIZZLE_128B atoms); a kernel's barriers and other control data follow its
// slots.  The producer waits on empty(s) with the opposite parity, fills the slot and
// completes full(s); the consumers wait on full(s) and each consumer warp arrives on
// empty(s) once it has finished reading.  `stage` / `phase` are the calling thread's
// position in the ring.
template <int S, int STAGE>
struct Ring {
  uint8_t* sm;                       // aligned start of dynamic shared memory
  uint32_t base, full0, empty0;      // shared addresses of slot 0, full(0), empty(0)
  int stage = 0, prev = -1;          // prev: slot of the consumer's k-block still in flight
  uint32_t phase = 0;

  __device__ __forceinline__ Ring(uint8_t* smem, uint32_t slots_off, uint32_t full_off,
                                  uint32_t empty_off) {
    const uint32_t raw = smem_u32(smem), a = (raw + 1023u) & ~1023u;
    sm = smem + (a - raw);
    base = a + slots_off;
    full0 = smem_u32(sm + full_off);
    empty0 = full0 + (empty_off - full_off);
  }
  __device__ __forceinline__ uint32_t stage_addr(int s) const { return base + s * STAGE; }
  __device__ __forceinline__ uint32_t full(int s) const { return full0 + 8u * s; }
  __device__ __forceinline__ uint32_t empty(int s) const { return empty0 + 8u * s; }
  // one thread, before the CTA barrier that publishes the ring
  __device__ __forceinline__ void init(uint32_t full_count, uint32_t empty_count) const {
    for (int s = 0; s < S; ++s) {
      mbar_init(full(s), full_count);
      mbar_init(empty(s), empty_count);
    }
    fence_barrier_init();
  }
  __device__ __forceinline__ void advance() {
    if (++stage == S) { stage = 0; phase ^= 1; }
  }

  // One k-block of a consumer warpgroup: wait for the slot, issue mma(stage address) as one
  // wgmma group, then wait for the PREVIOUS k-block's group and release its slot, so one
  // k-block stays in flight while the next is issued.
  template <int R, class MMA>
  __device__ __forceinline__ void consume(float (&acc)[R], MMA&& mma) {
    mbar_wait(full(stage), phase);
    fence_acc(acc);
    wgmma_fence();
    mma(stage_addr(stage));
    wgmma_commit();
    wgmma_wait<1>();
    fence_acc(acc);
    if (prev >= 0 && (threadIdx.x & 31) == 0) mbar_arrive(empty(prev));
    prev = stage;
    advance();
  }
  // end of a run of consume(): the last group completes and its slot is released
  template <int R>
  __device__ __forceinline__ void drain(float (&acc)[R]) {
    wgmma_wait<0>();
    fence_acc(acc);
    if (prev >= 0 && (threadIdx.x & 31) == 0) mbar_arrive(empty(prev));
    prev = -1;
  }
};

// ------------------------------------------------------------------ BatchNorm statistics
// The epilogues sum each output column and its square into a per-warp shared-memory slice
// [sum | sum of squares][BN]; a flush adds the slices in warp order, so the sums are
// identical run to run.
//
// Adds one fragment column pair cl, cl + 1: v[h][e] is row h (fragment rows r, r + 8) and
// column e; a row with ok[h] false counts as zero.  The eight lanes of a column are summed
// with shuffles and added to the slice by lanes 0-3.
template <int BN>
__device__ __forceinline__ void stats_add(float* wstat, int cl, const float (&v)[2][2],
                                          const bool (&ok)[2]) {
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const float x0 = ok[0] ? v[0][e] : 0.f, x1 = ok[1] ? v[1][e] : 0.f;
    float s1 = x0 + x1, s2 = fmaf(x0, x0, x1 * x1);
#pragma unroll
    for (int o = 4; o < 32; o <<= 1) {
      s1 += __shfl_xor_sync(0xffffffffu, s1, o);
      s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    if ((threadIdx.x & 31) < 4) {
      wstat[cl + e] += s1;
      wstat[BN + cl + e] += s2;
    }
  }
}
// Adds the slices of the WARPS consumer warps (thread t of 32 * WARPS, named barrier 1) in
// warp order into stats[sum | sum of squares][cout] for the columns of N tile nt below
// cout, one double atomic each, and zeroes the slices.
template <int BN, int WARPS>
__device__ __forceinline__ void stats_flush(float* sstat, int t, int nt, int cout,
                                            double* stats) {
  named_sync(1, 32 * WARPS);
  for (int c = t; c < 2 * BN; c += 32 * WARPS) {
    const int which = c / BN, col = nt * BN + (c % BN);
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < WARPS; ++w) {
      v += sstat[w * 2 * BN + c];
      sstat[w * 2 * BN + c] = 0.f;
    }
    if (col < cout) atomicAdd(stats + (int64_t)which * cout + col, (double)v);
  }
  named_sync(1, 32 * WARPS);
}

// round-to-nearest (ties away) TF32 kept in an fp32 container.  Same result as
// cvt.rna.tf32.f32 for finite inputs, in 2 integer instructions instead of the 4 the
// conversion expands to (it adds an Inf/NaN guard the operand split does not need).
__device__ __forceinline__ float to_tf32(float x) {
  return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xffffe000u);
}
// BatchNorm affine + optional ReLU of the producing layer (lb = 0 with ReLU, -inf without)
__device__ __forceinline__ float4 bn_act4(float4 x, float4 sc, float4 sh, float lb) {
  return make_float4(fmaxf(fmaf(x.x, sc.x, sh.x), lb), fmaxf(fmaf(x.y, sc.y, sh.y), lb),
                     fmaxf(fmaf(x.z, sc.z, sh.z), lb), fmaxf(fmaf(x.w, sc.w, sh.w), lb));
}

// ------------------------------------------------------------------ host: launch
// Launches Kernel with `smem` bytes of dynamic shared memory; the first call of each
// instantiation raises the kernel's dynamic shared-memory limit to it.
template <auto Kernel, class... Args>
int launch(unsigned grid, int threads, int smem, cudaStream_t st, const Args&... args) {
  static bool attr_set = false;
  if (!attr_set) {
    EPB_CUDA(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_set = true;
  }
  Kernel<<<grid, threads, smem, st>>>(args...);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

}  // namespace tc
