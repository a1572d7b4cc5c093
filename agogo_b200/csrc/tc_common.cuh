// agogo_b200 — shared pieces of the tensor-core kernels (tower_tc.cu: inference tower, train_tc.cu: training GEMMs):
// PTX wrappers (mbarrier, TMA, wgmma), shared-memory matrix descriptors, the implicit-GEMM 3x3 convolution kernel
// template and the host-side tensor-map builders.  Everything lives in an anonymous namespace: each translation unit
// instantiates what it launches.
//
// Hopper (sm_90a) structure of every GEMM kernel here: warp 8 (lane 0) is the TMA producer filling a ring of K-block
// stages (full/empty mbarriers); warps 0-7 are two consumer warpgroups, each owning 64 of the tile's 128 M rows and
// issuing wgmma.mma_async (m64 x BN x k16, both operands from shared memory, fp32 accumulators in registers), then
// running the epilogue straight from its registers while the producer already fills the next tile's stages.
// The number of tensor passes follows from the operand form at compile time (mma_kblock): a K block is one wgmma group
// with nothing between its wgmmas, so ptxas emits one warpgroup.arrive per block instead of fencing every wgmma.
// The fused layers' 192-row form (k_conv3x3_m192) runs the same body with three consumer warpgroups and no producer
// warp: lane 0 of warp 0 issues the loads between its own K blocks.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>

#include <cmath>
#include <cstdlib>
#include <cstring>
#include <stdexcept>

#include "mcts_dev.cuh"
#include "tower_tc.cuh"

namespace {


constexpr int BM = 128;        // M tile: two consumer warpgroups x 64 rows
constexpr int BK = 64;         // K block per pipeline stage: 64 fp16 = 128-byte rows (SWIZZLE_128B)
constexpr int NTHREADS = 288;  // warps 0-7: two consumer warpgroups; warp 8: TMA producer
constexpr int PRODUCER_WARP = 8;
constexpr int CONSUMER_WARPS = 8;
// k_conv3x3_m192: three consumer warpgroups x 64 rows, no producer warp (conv3x3_body)
constexpr int BM192 = 192;
constexpr int M192_THREADS = 384;
// H100: 227 KB of dynamic shared memory per block, less alignment slack and the barriers
constexpr int SMEM_RING_BUDGET = 227 * 1024 - 2048;
// OPS: fp16 planes stored per operand — 2 = hi/lo (fp32-faithful), 1 = one fp16 (AZ_FLAG_FP16_TOWER); bm: the M tile
__host__ __device__ constexpr int stage_bytes(int BN, int OPS = 2, int bm = BM) { return OPS * (bm * BK * 2 + BN * BK * 2); }
__host__ __device__ constexpr int num_stages(int BN, int OPS = 2, int bm = BM) {
  return SMEM_RING_BUDGET / stage_bytes(BN, OPS, bm) > 8 ? 8 : SMEM_RING_BUDGET / stage_bytes(BN, OPS, bm);
}
__host__ __device__ constexpr int smem_bytes(int BN, int OPS = 2, int bm = BM) {
  return num_stages(BN, OPS, bm) * stage_bytes(BN, OPS, bm) + 1024 + 256;
}
static_assert(num_stages(256, 2, BM192) == 2, "the 192-row fused tile double-buffers its 112 KB stages");

// The stored fp16 planes of an operand, and the tensor maps over them: hi and lo for the fp32-faithful form, hi alone for
// the fp16 form, so that a kernel instantiated for one plane has no lo to read or write.
template <int OPS> struct Planes { __half *hi, *lo; };
template <> struct Planes<1> { __half* hi; };
template <int OPS> struct PlaneMaps { CUtensorMap hi, lo; };
template <> struct PlaneMaps<1> { CUtensorMap hi; };

// The operand format of every tensor-core pass: v = hi + lo, hi = fp16(v), lo = fp16(v - hi).  Callers scale v by a
// power of two first so that lo stays a normal fp16.
__host__ __device__ __forceinline__ void split_hi_lo(float v, __half& hi, __half& lo) {
  hi = __float2half_rn(v);
  lo = __float2half_rn(v - __half2float(hi));
}

// ---------------------------------------------------------------------------------------------
// PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile(
        "{\n\t.reg .pred P;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, P;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
  } while (!ok);
}
// The stage ring of every kernel here: full[STAGES] then empty[STAGES] mbarriers at `bars`.  Pipeline step `it` uses
// stage it % STAGES in phase (it / STAGES) & 1.  The producer's lane waits until every consumer warp has released the
// stage's previous use, then arms full with the bytes its TMA loads will deliver; a consumer warp waits on full and,
// once its MMAs have read the stage, releases it with one arrival from lane 0.
template <int STAGES>
struct MbarRing {
  uint32_t bars;
  __device__ __forceinline__ static uint32_t stage(uint32_t it) { return it % STAGES; }
  __device__ __forceinline__ uint32_t full(uint32_t it) const { return bars + 8u * stage(it); }
  __device__ __forceinline__ uint32_t empty(uint32_t it) const { return bars + 8u * (STAGES + stage(it)); }
  __device__ __forceinline__ void init(uint32_t consumer_arrivals) const {  // by thread 0; the caller then __syncthreads
    if (threadIdx.x != 0) return;
    for (int s = 0; s < STAGES; s++) { mbar_init(full(s), 1); mbar_init(empty(s), consumer_arrivals); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __device__ __forceinline__ void producer_acquire(uint32_t it, uint32_t bytes) const {
    mbar_wait(empty(it), ((it / STAGES) & 1) ^ 1);
    mbar_expect_tx(full(it), bytes);
  }
  __device__ __forceinline__ void consumer_wait(uint32_t it) const {
    mbar_wait(full(it), (it / STAGES) & 1);
    __syncwarp();
  }
  __device__ __forceinline__ void consumer_release(uint32_t it) const {
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive(empty(it));
  }
};
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// im2col: consecutive pixels from (w, h, n) in W, H, N order over the map's bounding box, each read at (+dw, +dh);
// positions off the tensor read as zeros
__device__ __forceinline__ void tma_load_im2col(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c, int w, int h, int n,
                                                uint16_t dw, uint16_t dh) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2], "
      "{%7, %8};"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c), "r"(w), "r"(h), "r"(n), "h"(dw), "h"(dh)
      : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }// keeps the compiler from moving accumulator reads/writes across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; i++) asm volatile("" : "+f"(d[i])::"memory");
}

// D (+)= A[smem] * B[smem], m64 x N x k16, fp16 inputs, fp32 accumulate; TB = 1: B is MN-major (transposed)
template <int TB>
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
      "}, %32, %33, p, 1, 1, 0, %35;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate), "n"(TB));
}
template <int TB>
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
      "}, %64, %65, p, 1, 1, 0, %67;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate), "n"(TB));
}
template <int TB>
__device__ __forceinline__ void wgmma_n256(float (&d)[128], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
      "}, %128, %129, p, 1, 1, 0, %131;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate), "n"(TB));
}
template <int N, int TB>
__device__ __forceinline__ void wgmma_f16(float (&d)[N / 2], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  if constexpr (N == 256) wgmma_n256<TB>(d, desc_a, desc_b, accumulate);
  else if constexpr (N == 128) wgmma_n128<TB>(d, desc_a, desc_b, accumulate);
  else wgmma_n64<TB>(d, desc_a, desc_b, accumulate);
}

// wgmma shared-memory matrix descriptor: start >> 4 (bits 0-13) | LBO >> 4 (16-29) | SBO >> 4 (32-45) |
// layout type (bits 62-63: 1 = SWIZZLE_128B).  Tile bases are 1024-byte aligned, so the base offset (49-51) is 0.
// K-major, SWIZZLE_128B: rows of 64 fp16, 8-row atoms 1024 B apart (SBO); LBO unused.
__device__ __forceinline__ uint64_t make_desc_sw(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
// K-major, no swizzle: 8x16-byte core matrices, rows 16 B apart (8-row groups SBO = 128 B), 8-element K chunks lbo_bytes
// apart (canonical layout ((8,m),(T,2k)):((1T,SBO),(1,LBO)) in 16-byte units).  Any 16-byte-aligned start is valid, so a
// start `shift` rows into a tile is the same tile shifted by `shift` rows.
__device__ __forceinline__ uint64_t make_desc_plain(uint32_t smem_addr, uint32_t lbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)(lbo_bytes >> 4) << 16;
  d |= (uint64_t)(128 >> 4) << 32;
  return d;
}
// MN-major, SWIZZLE_128B: 64-element (128 B) runs along M/N, rows = K index; atoms of 8 K-rows (1024 B, SBO),
// 64-wide M/N groups lbo_bytes apart (canonical layout ((8,n),(8,k)):((1,LBO),(8,SBO)) in 16-byte units)
__device__ __forceinline__ uint64_t make_desc_mn_sw128(uint32_t smem_addr, uint32_t lbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)(lbo_bytes >> 4) << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// training operands carry a data-dependent power-of-two scale: the device word is max(ilogb(absmax) - 13, -127) (or the
// 0x80808080 fill when the tensor is all zero); scale exponent e = -word
__device__ __forceinline__ int exp_decode(const int* e) { const int v = *e; return v < -100000 ? 0 : -v; }
// v * 2^-e rounded once, as ldexpf(v, -e): one multiply while 2^-e is a normal float (e is the same for every thread, so
// the branch is uniform); ldexpf once 2^-e alone would flush to zero while the product is still a float
__device__ __forceinline__ float descale(float v, int e) {
  return e >= -127 && e <= 126 ? v * __int_as_float((127 - e) << 23) : ldexpf(v, -e);
}

struct ConvArgs {
  const int* n_dev;   // batch size (device)
  int n_max;
  int S, Wp, H, W;    // positions per sample (flat: (H+1)*(W+1), per-sample: H*(W+1)), row pitch W+1
  int guard;          // zero rows in front of the activation buffers (flat layout only)
  int mode3d, tps;    // per-sample layout: 3-D tensor map, tps = 128-row M tiles per sample
  int cin;            // padded input channels (multiple of 64)
  int n_total;        // GEMM N of the layer (fused: 2*K)
  int cout;           // output channels (K)
  const float2* aff;  // [HW][n_total] {A', B} in weight-row order
  float act_scale;    // 2^ea
  int* err;
  // raw mode (training, K7): no affine / ReLU / split — the epilogue writes acc * 2^-(*exp_a + *exp_b) as fp32
  float* out_raw;     // [(guard + rows)][n_total] or nullptr
  const int* exp_a;   // power-of-two scales of the A and B operands (device: they are data dependent)
  const int* exp_b;
};

// One K block of the product for this warpgroup's 64 rows: A rows at a_hi / a_lo, B (BN rows) at b_hi / b_lo.  The
// operand form sets the passes: OPS = 2 (hi/lo planes) runs hi*hi + hi*lo + lo*hi, fp32-faithful up to the dropped
// lo*lo; OPS = 1 (one fp16 plane) runs hi*hi alone and leaves the lo descriptors unused.
// a_step / b_step: descriptor start-address advance (16-byte units) per 16-wide K step.
template <int BN, int TB, int OPS = 2>
__device__ __forceinline__ void mma_kblock(float (&acc)[BN / 2], uint64_t dAh, uint64_t dAl, uint64_t dBh, uint64_t dBl,
                                           uint32_t b_step, bool first, uint32_t a_step = 32 >> 4) {
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < BK / 16; ks++) {
    const uint64_t adv = (uint64_t)ks * a_step;     // A: K-major SWIZZLE_128B: 16 fp16 = 32 B inside the atom
    const uint64_t advb = (uint64_t)ks * b_step;    // B: K-major as A; MN-major 16 K-rows of 128 B
    wgmma_f16<BN, TB>(acc, dAh + adv, dBh + advb, (first && ks == 0) ? 0u : 1u);
    if constexpr (OPS == 2) {
      wgmma_f16<BN, TB>(acc, dAh + adv, dBl + advb, 1u);
      wgmma_f16<BN, TB>(acc, dAl + adv, dBh + advb, 1u);
    }
  }
  wgmma_commit();
  wgmma_wait_all();
  acc_fence(acc);
}

// This consumer thread's place in its warpgroup's m64nNk16 accumulator fragment (warpgroup wg = warp / 4 owns tile rows
// wg*64 .. wg*64 + 63): acc[4j + 2h + e] = (tile row row0 + 8h, column 8j + col0 + e)
__device__ __forceinline__ void acc_frag_origin(int warp, int lane, int& row0, int& col0) {
  row0 = (warp >> 2) * 64 + (warp & 3) * 16 + (lane >> 2);
  col0 = 2 * (lane & 3);
}

// Output value of a fused layer at output column 8j + col0 + e of fragment row half h, before the hi/lo split: BN affine
// and ReLU, for a fused pair (PAIR) plus the second branch's, whose weight rows sit N/2 columns further in the tile, then
// the activation scale.  aff points at the tile's affine row of this position, offset by col0.
template <int N, bool PAIR>
__device__ __forceinline__ float fused_value(const float2* aff, const float (&acc)[N / 2], int j, int h, int e, float act_scale) {
  constexpr int OUTC = PAIR ? N / 2 : N;
  const float2 fa = __ldg(aff + 8 * j + e);
  float v = fmaxf(fmaf(fa.x, acc[4 * j + 2 * h + e], fa.y), 0.0f);
  if (PAIR) {
    const float2 fb = __ldg(aff + N / 2 + 8 * j + e);
    v += fmaxf(fmaf(fb.x, acc[4 * (j + OUTC / 8) + 2 * h + e], fb.y), 0.0f);
  }
  return v * act_scale;
}

// M tiles of a convolution over n samples for the kernel with WGS consumer warpgroups (64 * WGS rows per tile).  Per-sample
// layout: WGS = 3 tiles the n * H * W board points alone (im2col maps), WGS = 2 has whole 128-row tiles per sample.  Flat
// layout: tiles over the flat rows.
__host__ __device__ __forceinline__ int conv_m_tiles(const ConvArgs& a, int n, int WGS) {
  const int tm = 64 * WGS;
  if (WGS == 3 && a.mode3d) return (n * a.H * a.W + tm - 1) / tm;
  return a.mode3d ? n * a.tps : (n * a.S + tm - 1) / tm;
}

// The implicit-GEMM 3x3 convolution with WGS consumer warpgroups: an M tile of 64 * WGS rows.
//   WGS = 2 (288 threads): warp 8 is the TMA producer (lane 0 issues the loads).
//   WGS = 3 (384 threads): no producer warp.  A fourth warp would cap every thread at 152 registers (65536 / 416), and
//   one m64n256k16 wgmma with its 128 fp32 accumulators needs more; ptxas allocates the whole kernel under the launch
//   bound, so setmaxnreg cannot lend the consumers a producer warpgroup's registers either.  Lane 0 of warp 0 issues
//   the loads instead: STAGES steps ahead before the first K block, then step it + STAGES as soon as its own warp has
//   released step it.  It waits on the same empty barrier a producer warp would, so the loads start no later.
// OPS = 2: activations and filters as fp16 hi/lo planes (out: hi/lo, or raw fp32 for training).  OPS = 1: one fp16
// plane each, one pass, the output rounded once to fp16; half the bytes per stage, so a deeper ring.
// Stage layout: A planes, then B planes.
template <int WGS, int BN, bool PAIR, int OPS>
__device__ __forceinline__ void conv3x3_body(const PlaneMaps<OPS>& tmA, const PlaneMaps<OPS>& tmB, const ConvArgs& a,
                                             const Planes<OPS>& out) {
  static_assert(WGS == 2 || WGS == 3, "two or three consumer warpgroups");
  constexpr int TM = 64 * WGS;              // M tile
  constexpr int CONSUMERS = 4 * WGS;        // consumer warps (WGS = 2: the producer warp is the next one)
  constexpr int A_TILE_BYTES = TM * BK * 2;
  constexpr int STAGES = num_stages(BN, OPS, TM);
  constexpr int STAGE_BYTES = stage_bytes(BN, OPS, TM);
  constexpr int B_TILE_BYTES = BN * BK * 2;
  constexpr int OUTC = PAIR ? BN / 2 : BN;  // output channels per N tile
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const MbarRing<STAGES> ring{smem_base + STAGES * STAGE_BYTES};
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  ring.init(CONSUMERS);
  __syncthreads();

  const int n = min(*a.n_dev, a.n_max);
  const int rows = n * a.S;
  const int m_tiles = conv_m_tiles(a, n, WGS);
  const int n_tiles = a.n_total / BN;
  const int total_tiles = m_tiles * n_tiles;
  const int kc_per_tap = a.cin / BK;
  const int kblocks = 9 * kc_per_tap;

  // pipeline step `it`: wait until the stage is free, then TMA K block kb of M tile mt (first row m0), N tile from row n0
  const auto load_step = [&](uint32_t it, int mt, int m0, int n0, int kb) {
    ring.producer_acquire(it, STAGE_BYTES);
    const int tap = kb / kc_per_tap, kc = kb - tap * kc_per_tap;
    const int dy = tap / 3 - 1, dx = tap % 3 - 1;
    const uint32_t sa = smem_base + ring.stage(it) * STAGE_BYTES, bar = ring.full(it);
    if (WGS == 3 && a.mode3d) {
      // the tile's first board point (b, y, x); the map's pixels start at the window corner (x - 1, y - 1) and each
      // reads (+dx + 1, +dy + 1): tap (dy, dx), zero off the board
      const int HW = a.H * a.W, b = m0 / HW, q = m0 - b * HW, y = q / a.W, x = q - y * a.W;
      tma_load_im2col(sa, &tmA.hi, bar, kc * BK, x - 1, y - 1, b, (uint16_t)(dx + 1), (uint16_t)(dy + 1));
      if constexpr (OPS == 2)
        tma_load_im2col(sa + A_TILE_BYTES, &tmA.lo, bar, kc * BK, x - 1, y - 1, b, (uint16_t)(dx + 1), (uint16_t)(dy + 1));
    } else if (a.mode3d) {
      const int b = mt / a.tps, p0 = (mt - b * a.tps) * TM + dy * a.Wp + dx;  // may be <0 / >=S: zero fill
      tma_load_3d(sa, &tmA.hi, bar, kc * BK, p0, b);
      if constexpr (OPS == 2) tma_load_3d(sa + A_TILE_BYTES, &tmA.lo, bar, kc * BK, p0, b);
    } else {
      const int arow = a.guard + m0 + dy * a.Wp + dx;
      tma_load_2d(sa, &tmA.hi, bar, kc * BK, arow);
      if constexpr (OPS == 2) tma_load_2d(sa + A_TILE_BYTES, &tmA.lo, bar, kc * BK, arow);
    }
    tma_load_2d(sa + OPS * A_TILE_BYTES, &tmB.hi, bar, tap * a.cin + kc * BK, n0);
    if constexpr (OPS == 2) tma_load_2d(sa + 2 * A_TILE_BYTES + B_TILE_BYTES, &tmB.lo, bar, tap * a.cin + kc * BK, n0);
  };
  // WGS = 3: the loading lane's cursor over this CTA's (tile, K block) steps
  int p_tile = blockIdx.x, p_kb = 0;
  uint32_t p_it = 0;
  const auto load_next = [&]() {
    if (p_tile >= total_tiles) return;
    const int mt = p_tile / n_tiles;
    load_step(p_it++, mt, mt * TM, (p_tile - mt * n_tiles) * BN, p_kb);
    if (++p_kb == kblocks) { p_kb = 0; p_tile += gridDim.x; }
  };

  if constexpr (WGS == 2) {
    if (warp == CONSUMERS) {
      if (lane == 0) {
        // ===== TMA producer =====
        uint32_t it = 0;
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
          const int mt = tile / n_tiles, nt = tile - mt * n_tiles;
          const int m0 = mt * TM, n0 = nt * BN;
          for (int kb = 0; kb < kblocks; kb++, it++) load_step(it, mt, m0, n0, kb);
        }
      }
      return;
    }
  } else {
    if (threadIdx.x == 0)
      for (int s = 0; s < STAGES; s++) load_next();
  }
  // ===== consumer warpgroups 0 .. WGS-1: rows wg*64 .. wg*64+63 of the tile =====
  const int wg = warp >> 2;
  int row0, col0;
  acc_frag_origin(warp, lane, row0, col0);
  float acc[BN / 2];
  uint32_t it = 0;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const int mt = tile / n_tiles, nt = tile - mt * n_tiles;
    const int m0 = mt * TM, n0 = nt * BN;
    for (int kb = 0; kb < kblocks; kb++, it++) {
      ring.consumer_wait(it);
      const uint32_t sa = smem_base + ring.stage(it) * STAGE_BYTES;
      mma_kblock<BN, 0, OPS>(acc, make_desc_sw(sa + wg * 64 * 128), make_desc_sw(sa + A_TILE_BYTES + wg * 64 * 128),
                             make_desc_sw(sa + OPS * A_TILE_BYTES), make_desc_sw(sa + OPS * A_TILE_BYTES + B_TILE_BYTES), 32 >> 4,
                             kb == 0);
      ring.consumer_release(it);
      if constexpr (WGS == 3)
        if (threadIdx.x == 0) load_next();  // step it + STAGES, into the stage just released
    }
    // ===== epilogue from registers =====
    bool overflow = false;
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int lr = row0 + 8 * h;
      int r, p;  // r = row in the activation buffer (without guard), p = position inside the sample
      bool inb;
      if (WGS == 3 && a.mode3d) {  // row m0 + lr is board point q of sample b
        const int HW = a.H * a.W, pt = m0 + lr, b = pt / HW, q = pt - b * HW;
        p = q / a.W * a.Wp + q % a.W;
        r = b * a.S + p;
        inb = b < n;
      } else if (a.mode3d) {
        const int b = mt / a.tps;
        p = (mt - b * a.tps) * TM + lr;
        r = b * a.S + p;
        inb = p < a.S;
      } else {
        r = m0 + lr;
        p = r % a.S;
        inb = r < rows;
      }
      const int y = p / a.Wp, x = p - y * a.Wp;
      const bool valid = inb && y < a.H && x < a.W;
      if (!valid) continue;
      if constexpr (OPS == 2) {
        if (a.out_raw) {
          const int e = exp_decode(a.exp_a) + exp_decode(a.exp_b);
          float* o = a.out_raw + (size_t)(a.guard + r) * a.n_total + n0 + col0;
#pragma unroll
          for (int j = 0; j < BN / 8; j++)
            *reinterpret_cast<float2*>(o + 8 * j) = make_float2(descale(acc[4 * j + 2 * h], e), descale(acc[4 * j + 2 * h + 1], e));
          continue;
        }
      }
      const int hw = y * a.W + x;
      const float2* aff = a.aff + (size_t)hw * a.n_total + n0 + col0;
      const size_t o = (size_t)(a.guard + r) * a.cout + nt * OUTC + col0;
#pragma unroll
      for (int j = 0; j < OUTC / 8; j++) {
        __half hv[2], lv[2];
#pragma unroll
        for (int e = 0; e < 2; e++) {
          const float v = fused_value<BN, PAIR>(aff, acc, j, h, e, a.act_scale);
          if constexpr (OPS == 2) split_hi_lo(v, hv[e], lv[e]);
          else hv[e] = __float2half_rn(v);
          overflow |= !(fabsf(__half2float(hv[e])) <= 65504.0f);
        }
        *reinterpret_cast<__half2*>(out.hi + o + 8 * j) = __halves2half2(hv[0], hv[1]);
        if constexpr (OPS == 2) *reinterpret_cast<__half2*>(out.lo + o + 8 * j) = __halves2half2(lv[0], lv[1]);
      }
    }
    if (overflow) atomicOr(a.err, ERR_ACT_OVERFLOW);
  }
}

// 128-row tiles: every tower and training shape
template <int BN, bool PAIR, int OPS = 2>
__global__ void __launch_bounds__(NTHREADS, 1)
k_conv3x3_tc(const __grid_constant__ PlaneMaps<OPS> tmA, const __grid_constant__ PlaneMaps<OPS> tmB, ConvArgs a,
             Planes<OPS> out) {
  conv3x3_body<2, BN, PAIR, OPS>(tmA, tmB, a, out);
}
// 192-row tiles for the fused layers (hi/lo planes): 7/9 of the 128-row tile's operand bytes per MAC.  The activation
// maps have 192-row boxes.
template <int BN, bool PAIR>
__global__ void __launch_bounds__(M192_THREADS, 1)
k_conv3x3_m192(const __grid_constant__ PlaneMaps<2> tmA, const __grid_constant__ PlaneMaps<2> tmB, ConvArgs a, Planes<2> out) {
  conv3x3_body<3, BN, PAIR, 2>(tmA, tmB, a, out);
}

// The conv kernel with WGS consumer warpgroups, its block size and its dynamic shared memory
template <int WGS, int BN, bool PAIR, int OPS>
constexpr auto conv_kernel() {
  if constexpr (WGS == 2) return k_conv3x3_tc<BN, PAIR, OPS>;
  else return k_conv3x3_m192<BN, PAIR>;
}
constexpr int conv_threads(int WGS) { return WGS == 2 ? NTHREADS : M192_THREADS; }
constexpr int conv_smem_bytes(int WGS, int BN, int OPS) { return smem_bytes(BN, OPS, 64 * WGS); }

// dynamic shared memory opt-in of one instantiation on the current device (the attribute is per function and per device)
template <int WGS, int BN, bool PAIR, int OPS = 2>
void set_conv_attr() {
  CUDA_CHECK(cudaFuncSetAttribute(conv_kernel<WGS, BN, PAIR, OPS>(), cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  conv_smem_bytes(WGS, BN, OPS)));
}
// persistent grid: one CTA per SM, or one per tile when the largest batch has fewer
template <int WGS, int BN, bool PAIR, int OPS = 2>
void launch_conv(const PlaneMaps<OPS>& A, const PlaneMaps<OPS>& B, const ConvArgs& a, const Planes<OPS>& out, int num_sms,
                 cudaStream_t st) {
  const int grid = std::min(num_sms, conv_m_tiles(a, a.n_max, WGS) * (a.n_total / BN));
  const auto kernel = conv_kernel<WGS, BN, PAIR, OPS>();
  kernel<<<grid, conv_threads(WGS), conv_smem_bytes(WGS, BN, OPS), st>>>(A, B, a, out); LAUNCH_CHECK();
}

// ---------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q));
    if (!p || q != cudaDriverEntryPointSuccess) throw std::runtime_error("cuTensorMapEncodeTiled not available");
    fn = (EncodeTiledFn)p;
  }
  return fn;
}
// 2-D fp16 row-major [rows][cols] tensor, box {64 cols = 128 B, box_rows}, SWIZZLE_128B
CUtensorMap make_map(void* base, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  CUtensorMap m;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols * 2};
  cuuint32_t box[2] = {(cuuint32_t)BK, box_rows};
  cuuint32_t es[2] = {1, 1};
  CUresult r = get_encode()(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw std::runtime_error("cuTensorMapEncodeTiled failed: " + std::to_string((int)r));
  return m;
}

// per-sample layout: 3-D fp16 tensor [n][S][cols], box {64 cols, BM positions, 1 sample}
CUtensorMap make_map3d(void* base, uint64_t n, uint64_t S, uint64_t cols) {
  CUtensorMap m;
  cuuint64_t dims[3] = {cols, S, n};
  cuuint64_t strides[2] = {cols * 2, S * cols * 2};
  cuuint32_t box[3] = {(cuuint32_t)BK, (cuuint32_t)BM, 1};
  cuuint32_t es[3] = {1, 1, 1};
  CUresult r = get_encode()(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw std::runtime_error("cuTensorMapEncodeTiled(3d) failed: " + std::to_string((int)r));
  return m;
}

// per-sample layout seen as the board alone: 4-D fp16 tensor [n][H][W][cols] over the [n][H][W+1][cols] buffer (the zero
// column is skipped by the row stride), im2col boxes of `pixels` board points x 64 cols for a 3x3 window with padding 1:
// the bounding box runs from corner offset -1 to -1, so pixel (x, y) starts at window corner (x - 1, y - 1)
typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
CUtensorMap make_map_im2col(void* base, uint64_t n, uint64_t H, uint64_t W, uint64_t cols, uint32_t pixels) {
  static EncodeIm2colFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &p, cudaEnableDefault, &q));
    if (!p || q != cudaDriverEntryPointSuccess) throw std::runtime_error("cuTensorMapEncodeIm2col not available");
    fn = (EncodeIm2colFn)p;
  }
  CUtensorMap m;
  cuuint64_t dims[4] = {cols, W, H, n};
  cuuint64_t strides[3] = {cols * 2, (W + 1) * cols * 2, H * (W + 1) * cols * 2};
  int lower[2] = {-1, -1}, upper[2] = {-1, -1};
  cuuint32_t es[4] = {1, 1, 1, 1};
  CUresult r = fn(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, base, dims, strides, lower, upper, (cuuint32_t)BK, pixels, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw std::runtime_error("cuTensorMapEncodeIm2col failed: " + std::to_string((int)r));
  return m;
}

}  // namespace
