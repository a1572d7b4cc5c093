// agogo_b200 — K7 on tensor cores: the 3x3 convolutions of dual.Train (meta.go:16-54) as wgmma GEMMs (sm_90a).
// Forward and backward-data run through the tower's kernel (tc_common.cuh) in raw mode; both are the shifted-operand
// contraction
//   out[p, n] = sum_tap sum_k A[p + shift(tap), k] * Bm[n, tap*C + k]
// forward: A = x, Bm = filter;  backward-data: A = dz, Bm[ci, tap*Co + co] = filter[co][ci][8 - tap].
// Operands arrive as fp32 NCHW (the training pass keeps that layout); they are split into fp16 hi/lo
// at a data-dependent power-of-two scale (absmax -> exponent on device, gradients span many decades).
#include "tc_common.cuh"

namespace {

// K7 backward-filter on the same pipeline: dW[co][ci][tap] = sum_p dz[p, co] * x[p + shift(tap), ci].
// GEMM view: M = co, N = ci, K = board positions of the whole batch.  A = dz channel-major ([co][guard + positions],
// K-major).  B = x in the forward's position-major NHWC buffer, fed to the tensor core as an MN-major operand: the tap
// is a shift of the TMA ROW coordinate (a shift along the contiguous dimension would break TMA's 16-byte global
// alignment).  Work item = (tap, co tile, ci tile, K split); each item writes its fp32
// partial tile, k_dw_reduce sums the splits in a fixed order (deterministic, no atomics).
struct DwArgs {
  int co_tiles, ci_tiles, splits, kb_per_split;
  int guard, Wp, Co, Ci;
  float* partial;  // [splits][9][Co][Ci]
};
template <int BN>
__global__ void __launch_bounds__(NTHREADS, 1)
k_dw_tc(const __grid_constant__ CUtensorMap tmA_hi, const __grid_constant__ CUtensorMap tmA_lo,
        const __grid_constant__ CUtensorMap tmB_hi, const __grid_constant__ CUtensorMap tmB_lo, DwArgs a) {
  constexpr int A_TILE_BYTES = BM * BK * 2;
  constexpr int STAGES = num_stages(BN);
  constexpr int STAGE_BYTES = stage_bytes(BN);
  constexpr int B_TILE_BYTES = BN * BK * 2;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const MbarRing<STAGES> ring{smem_base + STAGES * STAGE_BYTES};
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  ring.init(CONSUMER_WARPS);
  __syncthreads();
  const int total_items = 9 * a.co_tiles * a.ci_tiles * a.splits;
  auto decode = [&](int item, int& tap, int& mt, int& nt, int& sp) {
    sp = item % a.splits; item /= a.splits;
    nt = item % a.ci_tiles; item /= a.ci_tiles;
    mt = item % a.co_tiles; tap = item / a.co_tiles;
  };
  if (warp == PRODUCER_WARP) {
    if (lane == 0) {
      uint32_t it = 0;
      for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
        int tap, mt, nt, sp;
        decode(item, tap, mt, nt, sp);
        const int shift = (tap / 3 - 1) * a.Wp + (tap % 3 - 1);
        for (int kb = 0; kb < a.kb_per_split; kb++, it++) {
          ring.producer_acquire(it, STAGE_BYTES);
          const uint32_t sa = smem_base + ring.stage(it) * STAGE_BYTES, bar = ring.full(it);
          const int col = a.guard + (sp * a.kb_per_split + kb) * BK;
          tma_load_2d(sa, &tmA_hi, bar, col, mt * BM);
          tma_load_2d(sa + A_TILE_BYTES, &tmA_lo, bar, col, mt * BM);
#pragma unroll
          for (int j = 0; j < BN / 64; j++) {  // [64 positions][64 channels] boxes, one per 64-wide N group
            tma_load_2d(sa + 2 * A_TILE_BYTES + j * 8192, &tmB_hi, bar, nt * BN + j * 64, col + shift);
            tma_load_2d(sa + 2 * A_TILE_BYTES + B_TILE_BYTES + j * 8192, &tmB_lo, bar, nt * BN + j * 64, col + shift);
          }
        }
      }
    }
    return;
  }
  const int wg = warp >> 2;
  int row0, col0;
  acc_frag_origin(warp, lane, row0, col0);
  float acc[BN / 2];
  uint32_t it = 0;
  for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
    int tap, mt, nt, sp;
    decode(item, tap, mt, nt, sp);
    for (int kb = 0; kb < a.kb_per_split; kb++, it++) {
      ring.consumer_wait(it);
      const uint32_t sa = smem_base + ring.stage(it) * STAGE_BYTES;
      // B operand MN-major: 16 K-rows of 128 B per k16 step
      mma_kblock<BN, 1>(acc, make_desc_sw(sa + wg * 64 * 128), make_desc_sw(sa + A_TILE_BYTES + wg * 64 * 128),
                        make_desc_mn_sw128(sa + 2 * A_TILE_BYTES, 8192), make_desc_mn_sw128(sa + 2 * A_TILE_BYTES + B_TILE_BYTES, 8192),
                        16 * 128 >> 4, kb == 0);
      ring.consumer_release(it);
    }
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int co = mt * BM + row0 + 8 * h;
      if (co >= a.Co) continue;
      float* o = a.partial + ((size_t)(sp * 9 + tap) * a.Co + co) * a.Ci + nt * BN + col0;
#pragma unroll
      for (int j = 0; j < BN / 8; j++) *reinterpret_cast<float2*>(o + 8 * j) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
    }
  }
}
// dW[co][ci][tap] = 2^-(ea+eb) * sum_split partial[split][tap][co][ci]
__global__ void k_dw_reduce(const float* __restrict__ partial, int splits, int Co, int Ci, const int* __restrict__ ea,
                            const int* __restrict__ eb, float* __restrict__ dW) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= Co * Ci) return;
  const int e = exp_decode(ea) + exp_decode(eb);
  const size_t tap_stride = (size_t)Co * Ci;
  for (int tap = 0; tap < 9; tap++) {
    float acc = 0.0f;
    for (int sp = 0; sp < splits; sp++) acc += partial[(size_t)(sp * 9 + tap) * tap_stride + idx];
    dW[(size_t)idx * 9 + tap] = descale(acc, e);
  }
}
// NCHW fp32 [B][C][HW] -> channel-major hi/lo [C][ld] at column guard + b*S + y*(W+1) + x, scaled by 2^(*exp)
__global__ void k_pack_cmajor(const float* __restrict__ x, int B, int C, int H, int W, int ld, int guard, int S,
                              const int* __restrict__ exp_in, __half* hi, __half* lo) {
  const int HW = H * W, Wp = W + 1;
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)B * C * HW) return;
  const int hw = (int)(idx % HW), c = (int)((idx / HW) % C), b = (int)(idx / ((size_t)HW * C));
  const int y = hw / W, xx = hw - y * W;
  const size_t o = (size_t)c * ld + guard + (size_t)b * S + y * Wp + xx;
  split_hi_lo(x[idx] * exp2f((float)exp_decode(exp_in)), hi[o], lo[o]);
}


__global__ void k_absmax_exp(const float* __restrict__ x, size_t n, int* exp_out) {
  __shared__ float sh[32];
  float m = 0.0f;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) m = fmaxf(m, fabsf(x[i]));
#pragma unroll
  for (int off = 16; off; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x < 32) {
    m = threadIdx.x < (blockDim.x >> 5) ? sh[threadIdx.x] : 0.0f;
#pragma unroll
    for (int off = 16; off; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
    // scale so that the largest magnitude lands in [2^13, 2^14): hi below fp16 overflow, lo as far from underflow as possible.
    // The scale 2^e must itself be a finite float (e <= 127): a tensor below 2^-114 lands lower, instead of 0 * inf = NaN.
    if (threadIdx.x == 0) atomicMax(exp_out, (m > 0.0f && isfinite(m)) ? max(ilogbf(m) - 13, -127) : -0x7fffffff);  // stores -e (max over blocks)
  }
}


// NCHW fp32 [B][C][HW] -> flat zero-bordered NHWC hi/lo [guard + B*S][cpad], scaled by 2^e.  Tile = 64 channels x
// 32 board points through shared memory: reads coalesced along hw, writes 128-byte runs along the channels.
__global__ void __launch_bounds__(256) k_pack_nchw(const float* __restrict__ x, int B, int C, int H, int W, int cpad, int guard, int S,
                                                   const int* __restrict__ exp_in, __half* hi, __half* lo) {
  __shared__ float t[64][33];
  const int HW = H * W, Wp = W + 1;
  const int hw0 = blockIdx.x * 32, c0 = blockIdx.y * 64, b = blockIdx.z;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  const float sc = exp2f((float)exp_decode(exp_in));
#pragma unroll
  for (int i = 0; i < 8; i++) {
    const int c = c0 + ty + 8 * i, hw = hw0 + tx;
    t[ty + 8 * i][tx] = (c < C && hw < HW) ? x[((size_t)b * C + c) * HW + hw] * sc : 0.0f;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int hw = hw0 + ty + 8 * i;
    if (hw >= HW) continue;
    const int y = hw / W, xx = hw - y * W;
    const size_t o = ((size_t)guard + (size_t)b * S + y * Wp + xx) * cpad + c0 + 2 * tx;
    __half h0, l0, h1, l1;
    split_hi_lo(t[2 * tx][ty + 8 * i], h0, l0);
    split_hi_lo(t[2 * tx + 1][ty + 8 * i], h1, l1);
    *reinterpret_cast<__half2*>(hi + o) = __halves2half2(h0, h1);
    *reinterpret_cast<__half2*>(lo + o) = __halves2half2(l0, l1);
  }
}
// flat NHWC fp32 [guard + B*S][ld] -> NCHW [B][C][HW] (assign or accumulate); 32 x 32 tiles through shared memory
__global__ void __launch_bounds__(256) k_unpack_nchw(const float* __restrict__ raw, int B, int C, int H, int W, int ld, int guard, int S,
                                                     float* out, int accumulate) {
  __shared__ float t[32][33];
  const int HW = H * W, Wp = W + 1;
  const int hw0 = blockIdx.x * 32, c0 = blockIdx.y * 32, b = blockIdx.z;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int hw = hw0 + ty + 8 * i, c = c0 + tx;
    float v = 0.0f;
    if (hw < HW && c < C) { const int y = hw / W, xx = hw - y * W; v = raw[((size_t)guard + (size_t)b * S + y * Wp + xx) * ld + c]; }
    t[ty + 8 * i][tx] = v;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int c = c0 + ty + 8 * i, hw = hw0 + tx;
    if (c < C && hw < HW) {
      const size_t o = ((size_t)b * C + c) * HW + hw;
      if (accumulate) out[o] += t[tx][ty + 8 * i]; else out[o] = t[tx][ty + 8 * i];
    }
  }
}
// filter [Co][Ci][3][3] -> Bm hi/lo [rows][9*cpad]; flip = backward-data operand (rows = Ci, K = tap*Co + co, mirrored taps)
__global__ void k_prep_filter(const float* __restrict__ w, int Co, int Ci, int cpad, int flip, const int* __restrict__ exp_in,
                              __half* hi, __half* lo) {
  const int rows = flip ? Ci : Co, kin = flip ? Co : Ci;
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)rows * 9 * cpad) return;
  const int kc = (int)(idx % cpad), tap = (int)((idx / cpad) % 9), row = (int)(idx / ((size_t)9 * cpad));
  float v = 0.0f;
  if (kc < kin) v = flip ? w[((size_t)kc * Ci + row) * 9 + (8 - tap)] : w[((size_t)row * Ci + kc) * 9 + tap];
  split_hi_lo(v * exp2f((float)exp_decode(exp_in)), hi[idx], lo[idx]);
}

// dynamic shared memory opt-in of the instantiations this file launches (per function, per device)
void train_configure_device() {
  set_conv_attr<2, 256, false>(); set_conv_attr<2, 128, false>(); set_conv_attr<2, 64, false>();
  CUDA_CHECK(cudaFuncSetAttribute(k_dw_tc<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes(256)));
  CUDA_CHECK(cudaFuncSetAttribute(k_dw_tc<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes(128)));
  CUDA_CHECK(cudaFuncSetAttribute(k_dw_tc<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes(64)));
}

}  // namespace


struct TcGemmImpl {
  NetDims d;
  int B, guard, S, rows_alloc, num_sms, cmax;
  // Two position-major (NHWC, zero-bordered) fp16 hi/lo operand slots [(rows)][cmax] with their power-of-two exponents:
  // slot 0 holds activations x (forward A operand, backward-filter B operand), slot 1 holds gradients dz (backward-data
  // A operand).  Keeping them apart lets the two branches of a block share one pack of x, and the backward-filter and
  // backward-data passes of a unit share one absmax of dz.
  struct Slot {
    __half *hi = nullptr, *lo = nullptr;
    int* exp = nullptr;
    int cpad = 0;  // channel pitch the buffers currently hold (their zero borders are only valid for that pitch)
  } slot[2];
  __half *w_hi = nullptr, *w_lo = nullptr;  // B operand [cmax][9*cmax]
  float* raw = nullptr;                     // [(rows)][cmax]
  int *exp_b = nullptr, *dB = nullptr;
  // backward-filter A operand (dz), channel-major [max(K,128)][ld], scaled by slot[1].exp
  __half *t_hi = nullptr, *t_lo = nullptr;
  float* partial = nullptr;
  int ld = 0, splits = 1, kb_per_split = 0, crow = 0;
};

bool tc_gemm_supported(const NetDims& d) { return d.K == 64 || d.K == 128 || d.K == 256; }

void tc_gemm_create(TcGemm& g, const NetDims& d, int B) {
  train_configure_device();
  TcGemmImpl* I = new TcGemmImpl;
  g.impl = I;
  I->d = d; I->B = B;
  I->guard = ((d.W + 2 + 7) / 8) * 8;
  I->S = (d.H + 1) * (d.W + 1);
  I->rows_alloc = I->guard + B * I->S + I->guard + BM;
  I->cmax = d.K;
  int dev;
  CUDA_CHECK(cudaGetDevice(&dev));
  CUDA_CHECK(cudaDeviceGetAttribute(&I->num_sms, cudaDevAttrMultiProcessorCount, dev));
  auto alloc_h = [&](size_t n) { __half* p; CUDA_CHECK(cudaMalloc(&p, n * 2)); CUDA_CHECK(cudaMemset(p, 0, n * 2)); return p; };
  for (auto& sl : I->slot) {
    sl.hi = alloc_h((size_t)I->rows_alloc * I->cmax); sl.lo = alloc_h((size_t)I->rows_alloc * I->cmax);
    CUDA_CHECK(cudaMalloc(&sl.exp, 4));
  }
  I->w_hi = alloc_h((size_t)I->cmax * 9 * I->cmax); I->w_lo = alloc_h((size_t)I->cmax * 9 * I->cmax);
  CUDA_CHECK(cudaMalloc(&I->raw, (size_t)I->rows_alloc * I->cmax * 4));
  CUDA_CHECK(cudaMalloc(&I->exp_b, 4)); CUDA_CHECK(cudaMalloc(&I->dB, 4));
  CUDA_CHECK(cudaMemcpy(I->dB, &B, 4, cudaMemcpyHostToDevice));
  // backward-filter: K = positions, split so that 9 * tiles * splits fills the SMs once
  {
    const int bn = std::min(256, d.K), tiles = ((d.K + BM - 1) / BM) * (d.K / bn);
    const int kb_total = (B * I->S + 63) / 64;
    I->splits = std::max(1, std::min(kb_total, I->num_sms / (9 * tiles)));
    I->kb_per_split = (kb_total + I->splits - 1) / I->splits;
    I->ld = I->guard + I->splits * I->kb_per_split * 64 + I->guard + 64;
    I->crow = std::max(d.K, BM);
    I->t_hi = alloc_h((size_t)I->crow * I->ld); I->t_lo = alloc_h((size_t)I->crow * I->ld);
    CUDA_CHECK(cudaMalloc(&I->partial, (size_t)I->splits * 9 * d.K * d.K * 4));
  }
}
void tc_gemm_destroy(TcGemm& g) {
  TcGemmImpl* I = (TcGemmImpl*)g.impl;
  if (!I) return;
  for (auto& sl : I->slot) { cudaFree(sl.hi); cudaFree(sl.lo); cudaFree(sl.exp); }
  cudaFree(I->w_hi); cudaFree(I->w_lo); cudaFree(I->raw);
  cudaFree(I->exp_b); cudaFree(I->dB);
  cudaFree(I->t_hi); cudaFree(I->t_lo); cudaFree(I->partial);
  delete I;
  g.impl = nullptr;
}

static void absmax_exp(const float* x, size_t n, int* e, cudaStream_t st) {
  CUDA_CHECK(cudaMemsetAsync(e, 0x80, 4, st));  // 0x80808080: below every real exponent
  unsigned blocks = (unsigned)std::min<size_t>((n + 1023) / 1024, 1024);
  k_absmax_exp<<<blocks, 256, 0, st>>>(x, n, e); LAUNCH_CHECK();
}

// Brings the NCHW tensor x [B][C][HW] into operand slot `si` according to `state`; returns the number of kernels launched.
static int fill_slot(TcGemmImpl* I, int si, const float* x, int C, int state, cudaStream_t st) {
  if (state == TC_OPERAND_REUSE) return 0;
  const NetDims& d = I->d;
  TcGemmImpl::Slot& sl = I->slot[si];
  const int cpad = (C + 63) & ~63;  // K-chunk granularity of the kernel
  if (sl.cpad != cpad) {
    CUDA_CHECK(cudaMemsetAsync(sl.hi, 0, (size_t)I->rows_alloc * I->cmax * 2, st));
    CUDA_CHECK(cudaMemsetAsync(sl.lo, 0, (size_t)I->rows_alloc * I->cmax * 2, st));
    sl.cpad = cpad;
  }
  int n = 1;
  if (state == TC_OPERAND_PACK) { absmax_exp(x, (size_t)I->B * C * d.HW(), sl.exp, st); n++; }
  k_pack_nchw<<<dim3((d.HW() + 31) / 32, cpad / 64, I->B), 256, 0, st>>>(x, I->B, C, d.H, d.W, cpad, I->guard, I->S, sl.exp, sl.hi, sl.lo); LAUNCH_CHECK();
  return n;
}

// out (NCHW [B][Cout][HW]) (+)= conv3x3(x (NCHW [B][Cin][HW]), filter [Co][Ci][3][3]) or its backward-data twin.
// x goes through operand slot a_slot (0: activations, 1: gradients) according to a_state.
void tc_gemm_conv(TcGemm& g, const float* x, int Cin, const float* filter, int fCo, int fCi, bool flip, float* out, int Cout,
                  bool accumulate, int a_slot, int a_state, cudaStream_t st, unsigned long long* launches) {
  TcGemmImpl* I = (TcGemmImpl*)g.impl;
  const NetDims& d = I->d;
  const int HW = d.HW();
  const int cpad = (Cin + 63) & ~63;
  if (cpad > I->cmax || Cout > I->cmax || (Cout % 64) != 0) throw std::runtime_error("tc_gemm_conv: unsupported channel count");
  TcGemmImpl::Slot& sl = I->slot[a_slot];
  if (a_state == TC_OPERAND_REUSE && sl.cpad != cpad) throw std::runtime_error("tc_gemm_conv: operand slot does not hold this shape");
  int nl = fill_slot(I, a_slot, x, Cin, a_state, st);
  absmax_exp(filter, (size_t)fCo * fCi * 9, I->exp_b, st);
  {
    size_t wt = (size_t)Cout * 9 * cpad;
    k_prep_filter<<<(unsigned)((wt + 255) / 256), 256, 0, st>>>(filter, fCo, fCi, cpad, flip ? 1 : 0, I->exp_b, I->w_hi, I->w_lo); LAUNCH_CHECK();
  }
  const int bn = std::min(256, Cout);
  // tensor maps over the (re-used) operand buffers for this shape
  const PlaneMaps<2> mA{make_map(sl.hi, I->rows_alloc, cpad, BM), make_map(sl.lo, I->rows_alloc, cpad, BM)};
  const PlaneMaps<2> mB{make_map(I->w_hi, Cout, (uint64_t)9 * cpad, bn), make_map(I->w_lo, Cout, (uint64_t)9 * cpad, bn)};
  ConvArgs a;
  a.n_dev = I->dB; a.n_max = I->B; a.S = I->S; a.Wp = d.W + 1; a.H = d.H; a.W = d.W; a.guard = I->guard; a.mode3d = 0; a.tps = 1;
  a.cin = cpad; a.n_total = Cout; a.cout = Cout; a.aff = nullptr; a.act_scale = 1.0f;
  a.err = nullptr; a.out_raw = I->raw; a.exp_a = sl.exp; a.exp_b = I->exp_b;
  const Planes<2> none{nullptr, nullptr};  // raw mode: the epilogue writes out_raw
  if (bn == 256) launch_conv<2, 256, false>(mA, mB, a, none, I->num_sms, st);
  else if (bn == 128) launch_conv<2, 128, false>(mA, mB, a, none, I->num_sms, st);
  else launch_conv<2, 64, false>(mA, mB, a, none, I->num_sms, st);
  k_unpack_nchw<<<dim3((HW + 31) / 32, (Cout + 31) / 32, I->B), 256, 0, st>>>(I->raw, I->B, Cout, d.H, d.W, Cout, I->guard, I->S, out, accumulate ? 1 : 0); LAUNCH_CHECK();
  if (launches) *launches += nl + 4;
}

// dW[K][K][3][3] = backward-filter of a K->K 3x3 layer for x (NCHW [B][K][HW]) and dz (NCHW [B][K][HW]).
// x goes through slot 0 according to x_state; the exponent of dz is left in slot 1 (a following backward-data call on the
// same dz passes TC_OPERAND_PACK_KEEP_EXP).
void tc_gemm_dw(TcGemm& g, const float* x, const float* dz, float* dW, int x_state, cudaStream_t st, unsigned long long* launches) {
  TcGemmImpl* I = (TcGemmImpl*)g.impl;
  const NetDims& d = I->d;
  const int C = d.K, HW = d.HW();
  const size_t n = (size_t)I->B * C * HW;
  TcGemmImpl::Slot& sx = I->slot[0];
  if (x_state == TC_OPERAND_REUSE && sx.cpad != C) throw std::runtime_error("tc_gemm_dw: operand slot does not hold this shape");
  int nl = fill_slot(I, 0, x, C, x_state, st);
  int* exp_dz = I->slot[1].exp;
  absmax_exp(dz, n, exp_dz, st);
  k_pack_cmajor<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(dz, I->B, C, d.H, d.W, I->ld, I->guard, I->S, exp_dz, I->t_hi, I->t_lo); LAUNCH_CHECK();
  const int bn = std::min(256, C);
  CUtensorMap mAh = make_map(I->t_hi, I->crow, I->ld, BM), mAl = make_map(I->t_lo, I->crow, I->ld, BM);
  CUtensorMap mBh = make_map(sx.hi, I->rows_alloc, C, 64), mBl = make_map(sx.lo, I->rows_alloc, C, 64);
  DwArgs a;
  a.co_tiles = (C + BM - 1) / BM; a.ci_tiles = C / bn; a.splits = I->splits; a.kb_per_split = I->kb_per_split;
  a.guard = I->guard; a.Wp = d.W + 1; a.Co = C; a.Ci = C; a.partial = I->partial;
  const int items = 9 * a.co_tiles * a.ci_tiles * a.splits;
  const int grid = std::min(I->num_sms, items);
  auto launch = [&](auto kern, int BNv) {
    kern<<<grid, NTHREADS, smem_bytes(BNv), st>>>(mAh, mAl, mBh, mBl, a); LAUNCH_CHECK();
  };
  if (bn == 256) launch(k_dw_tc<256>, 256);
  else if (bn == 128) launch(k_dw_tc<128>, 128);
  else launch(k_dw_tc<64>, 64);
  k_dw_reduce<<<(C * C + 255) / 256, 256, 0, st>>>(I->partial, I->splits, C, C, exp_dz, sx.exp, dW); LAUNCH_CHECK();
  if (launches) *launches += nl + 4;
}
