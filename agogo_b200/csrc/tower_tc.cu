// agogo_b200 — K5: the residual tower as wgmma / TMA implicit GEMMs (sm_90a).
//
// One kernel launch per conv layer (the init 3x3 conv, then one launch per shared block computing
// BOTH parallel branches as a single C->2C contraction, dualnet/dual.go:59-73):
//   out[p, c] = relu(Aa[hw,c]*convA(x)[p,c] + Ba[hw,c]) + relu(Ab[hw,c]*convB(x)[p,c] + Bb[hw,c])
// GEMM view: M = padded board positions of the whole batch, N = output channels, K = 9 taps x C_in.
//   * activations live in HBM as NHWC fp16 hi/lo planes over a zero-bordered position grid
//     ((H+1) x (W+1) per sample: one shared zero column / zero row), so that tap (dy,dx) of an
//     M-tile is the SAME 2-D TMA box shifted by dy*(W+1)+dx rows — im2col by TMA coordinates,
//     no gather, halo = zeros already in memory (or TMA out-of-bounds zero fill).  Two position
//     layouts, chosen per board size by padded-row overhead: "flat" = (H+1)x(W+1) positions per
//     sample, samples back to back, 2-D tensor map (9x9: 100/81); "per-sample" = Hx(W+1) positions,
//     3-D tensor map [sample][position][channel] whose out-of-range positions are zero-filled by
//     TMA, M-tiles never straddle samples (19x19: 3 tiles = 384 rows per 361 points vs 400);
//   * fp32 fidelity on fp16 tensor cores: x = hi + lo and w = hi + lo (both pre-scaled by powers of
//     two), three wgmma passes per K-step (hi*hi + hi*lo + lo*hi) into one fp32 register
//     accumulator; the dropped lo*lo term is ~2^-22 relative;
//   * warp roles (tc_common.cuh): one TMA producer warp, two consumer warpgroups of 64 rows each;
//     smem ring of K-blocks (full/empty mbarriers), persistent CTAs striding over (M-tile, N-tile),
//     epilogue (BN-affine + ReLU + branch add -> fp16 hi/lo split -> global) from the accumulators.
// Descriptor bit layouts follow the PTX ISA "Matrix Descriptor Format" table of wgmma.
#include "tc_common.cuh"

namespace {

// the first layer's input at (sample b, channel c, board point hw) before the hi/lo split: the scaled encoder plane, zero
// off the board and in the channels padded beyond F (k_pack_planes and k_net_small write the same operand)
__device__ __forceinline__ float plane_input(const float* planes, int F, int HW, int b, int c, int hw, bool on_board, float scale) {
  return on_board && c < F ? planes[((size_t)b * F + c) * HW + hw] * scale : 0.0f;
}

// fp32 NCHW planes -> zero-bordered NHWC fp16 hi/lo (channels padded to cpad)
__global__ void k_pack_planes(const float* __restrict__ planes, const int* __restrict__ n_dev, int n_max, int F, int H,
                              int W, int cpad, int guard, int S, float scale, __half* hi, __half* lo) {
  const int n = min(*n_dev, n_max);
  const int HW = H * W, Wp = W + 1;
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)n * HW * cpad) return;
  const int c = (int)(idx % cpad);
  const int hw = (int)((idx / cpad) % HW);
  const int b = (int)(idx / ((size_t)cpad * HW));
  const int y = hw / W, x = hw - y * W;
  __half h, l;
  split_hi_lo(plane_input(planes, F, HW, b, c, hw, true, scale), h, l);
  const size_t o = ((size_t)guard + (size_t)b * S + y * Wp + x) * cpad + c;
  hi[o] = h;
  lo[o] = l;
}
// The two 1x1 head convs (K->2 policy, K->1 value; dual.go:70,85) + BN-test affine + ReLU straight
// from the tower's NHWC hi/lo output: one warp per board point, lanes split the channels
// (coalesced 16-byte loads), three dot products reduced with shuffles.
//   ph [n][2][HW], vh [n][HW]  (the layout the linear layers consume)
__global__ void k_head_convs_nhwc(const __half* __restrict__ hi, const __half* __restrict__ lo, const int* __restrict__ n_dev,
                                  int n_max, int K, int H, int W, int guard, int S, float inv_scale, const float* __restrict__ wp,
                                  const float* __restrict__ gp, const float* __restrict__ bp, const float* __restrict__ wv,
                                  const float* __restrict__ gv, const float* __restrict__ bv, float* ph, float* vh) {
  const int n = min(*n_dev, n_max);
  const int HW = H * W, Wp = W + 1;
  const int lane = threadIdx.x & 31;
  const size_t wid = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (wid >= (size_t)n * HW) return;
  const int b = (int)(wid / HW), hw = (int)(wid - (size_t)b * HW);
  const int y = hw / W, x = hw - y * W;
  const size_t row = (size_t)guard + (size_t)b * S + y * Wp + x;
  float a0 = 0.0f, a1 = 0.0f, a2 = 0.0f;
  for (int c0 = lane * 8; c0 < K; c0 += 256) {
    const uint4 h4 = *(const uint4*)(hi + row * K + c0);
    const uint4 l4 = *(const uint4*)(lo + row * K + c0);
    const __half* hh = (const __half*)&h4;
    const __half* ll = (const __half*)&l4;
#pragma unroll
    for (int i = 0; i < 8; i++) {
      const float v = (__half2float(hh[i]) + __half2float(ll[i])) * inv_scale;
      a0 = fmaf(v, __ldg(wp + c0 + i), a0);
      a1 = fmaf(v, __ldg(wp + K + c0 + i), a1);
      a2 = fmaf(v, __ldg(wv + c0 + i), a2);
    }
  }
#pragma unroll
  for (int off = 16; off; off >>= 1) {
    a0 += __shfl_xor_sync(0xffffffffu, a0, off);
    a1 += __shfl_xor_sync(0xffffffffu, a1, off);
    a2 += __shfl_xor_sync(0xffffffffu, a2, off);
  }
  if (lane == 0) {
    const float isd = 1.0f / sqrtf(1e-5f);
    float p0 = gp[hw] * (a0 * isd) + bp[hw];
    float p1 = gp[HW + hw] * (a1 * isd) + bp[HW + hw];
    float v0 = gv[hw] * (a2 * isd) + bv[hw];
    ph[((size_t)b * 2 + 0) * HW + hw] = p0 > 0.0f ? p0 : 0.0f;
    ph[((size_t)b * 2 + 1) * HW + hw] = p1 > 0.0f ? p1 : 0.0f;
    vh[(size_t)b * HW + hw] = v0 > 0.0f ? v0 : 0.0f;
  }
}
// diagnostics: the NHWC hi/lo tower output (the values k_head_convs_nhwc reads) -> fp32 NCHW [n][K][HW]
__global__ void k_tower_nchw(const __half* __restrict__ hi, const __half* __restrict__ lo, const int* __restrict__ n_dev, int n_max,
                             int K, int H, int W, int guard, int S, float inv_scale, float* out) {
  const int n = min(*n_dev, n_max);
  const int HW = H * W, Wp = W + 1;
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)n * K * HW) return;
  const int hw = (int)(idx % HW), c = (int)((idx / HW) % K), b = (int)(idx / ((size_t)HW * K));
  const int y = hw / W, x = hw - y * W;
  const size_t o = ((size_t)guard + (size_t)b * S + y * Wp + x) * K + c;
  out[idx] = (__half2float(hi[o]) + __half2float(lo[o])) * inv_scale;
}

// -------------------------------------------------------------------------------------------------
// k_net_small: the whole tower of a K = 64 net on a board of at most 128 padded positions ((H+1)(W+1) <= 128, BASELINE
// C2) in one persistent kernel.  A 3x3 convolution mixes board points of one sample only, so a CTA carries a sample
// through every layer with no grid-wide step: the sample's zero-bordered positions x 64 channels stay in shared memory as
// fp16 hi / lo planes (two ping-pong buffers), only the filters stream from L2 (TMA into an mbarrier ring that runs ahead
// across layers and samples, one stage per (layer, tap)), and the last layer writes the NHWC hi/lo buffer the head
// kernels read.  Activations are stored K-major without swizzle ([8-channel chunk][row][16 B]), so tap (dy, dx) is the
// same tile with its descriptor starting dy*(W+1)+dx rows further — no copy per tap.  Same MMA sequence (tap by tap, three
// passes), same epilogue arithmetic as the per-layer kernels: the outputs are identical to that path.
constexpr int SN_MAXL = 8;                 // init conv + up to 7 blocks
constexpr int SN_R0 = 16;                  // halo rows in front of the tile (>= W + 2)
constexpr int SN_HR = 160;                 // rows per activation plane: halo + 128 + halo
constexpr int SN_PLANE = 8 * SN_HR * 16;   // one fp16 plane: 8 chunks of 8 channels x SN_HR rows x 16 B
constexpr int SN_NST = 4;                  // filter stages
constexpr int SN_STAGE = 2 * 128 * BK * 2; // hi + lo filter tiles of up to 128 rows x 64 K
__host__ __device__ constexpr int smem_bytes_small() { return 4 * SN_PLANE + SN_NST * SN_STAGE + 1024 + 256; }
struct SmallMaps { CUtensorMap hi[SN_MAXL], lo[SN_MAXL]; };
struct SmallNetArgs {
  const float* planes;  // [n][F][HW] encoder planes
  const int* n_dev;
  int n_max, F, H, W, Wp, S, HW, nlayers, guard;
  float act_scale;
  const float2* aff[SN_MAXL];  // per layer [HW][n_total] {A', B}
  __half *out_hi, *out_lo;     // last layer: [(guard + n*S)][64], the layout k_head_convs_nhwc reads
  int* err;
};

// one layer of one sample: 9 taps of the filter ring into acc, then the epilogue into smem (or global for the last layer)
template <int N>
__device__ __forceinline__ void small_layer(const SmallNetArgs& a, int l, int smp, uint32_t act, uint32_t stages,
                                            const MbarRing<SN_NST>& ring, uint32_t& it, int in, bool& overflow) {
  constexpr bool PAIR = N == 128;
  constexpr int OUTC = PAIR ? N / 2 : N;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
  int row0, col0;
  acc_frag_origin(warp, lane, row0, col0);
  const uint32_t in_hi = act + (2 * in) * SN_PLANE, in_lo = in_hi + SN_PLANE;
  float acc[N / 2];
  for (int tap = 0; tap < 9; tap++, it++) {
    ring.consumer_wait(it);
    const uint32_t shift = (uint32_t)(SN_R0 + wg * 64 + (tap / 3 - 1) * a.Wp + (tap % 3 - 1)) * 16;
    const uint32_t sb = stages + ring.stage(it) * SN_STAGE;
    mma_kblock<N, 0>(acc, make_desc_plain(in_hi + shift, SN_HR * 16), make_desc_plain(in_lo + shift, SN_HR * 16),
                     make_desc_sw(sb), make_desc_sw(sb + SN_STAGE / 2), 32 >> 4, tap == 0, 2 * SN_HR * 16 >> 4);
    ring.consumer_release(it);
  }
  const bool last = l == a.nlayers - 1;
  const uint32_t out_hi = act + (2 * (in ^ 1)) * SN_PLANE, out_lo = out_hi + SN_PLANE;
  const int n_total = PAIR ? 128 : 64;
#pragma unroll
  for (int h = 0; h < 2; h++) {
    const int p = row0 + 8 * h;  // position inside the sample
    const int y = p / a.Wp, x = p - y * a.Wp;
    const bool valid = p < a.S && y < a.H && x < a.W;
    if (last && !valid) continue;
    const float2* aff = a.aff[l] + (size_t)(valid ? y * a.W + x : 0) * n_total + col0;
    const size_t grow = (size_t)a.guard + (size_t)smp * a.S + p;
#pragma unroll
    for (int j = 0; j < OUTC / 8; j++) {
      __half hv[2], lv[2];
#pragma unroll
      for (int e = 0; e < 2; e++) {
        split_hi_lo(valid ? fused_value<N, PAIR>(aff, acc, j, h, e, a.act_scale) : 0.0f, hv[e], lv[e]);
        overflow |= !(fabsf(__half2float(hv[e])) <= 65504.0f);
      }
      const int c = 8 * j + col0;
      if (last) {
        *reinterpret_cast<__half2*>(a.out_hi + grow * 64 + c) = __halves2half2(hv[0], hv[1]);
        *reinterpret_cast<__half2*>(a.out_lo + grow * 64 + c) = __halves2half2(lv[0], lv[1]);
      } else {  // chunk c / 8, row SN_R0 + p, byte (c % 8) * 2; invalid positions are written as zeros
        const uint32_t o = (uint32_t)(c >> 3) * (SN_HR * 16) + (uint32_t)(SN_R0 + p) * 16 + (uint32_t)(c & 7) * 2;
        const __half2 h2 = __halves2half2(hv[0], hv[1]), l2 = __halves2half2(lv[0], lv[1]);
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(out_hi + o), "r"(*reinterpret_cast<const uint32_t*>(&h2)) : "memory");
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(out_lo + o), "r"(*reinterpret_cast<const uint32_t*>(&l2)) : "memory");
      }
    }
  }
}

__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }
__device__ __forceinline__ void proxy_fence() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__global__ void __launch_bounds__(NTHREADS, 1) k_net_small(const __grid_constant__ SmallMaps maps, SmallNetArgs a) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* base_ptr = smem_raw + (base - smem_u32(smem_raw));
  const uint32_t act = base;                       // 4 planes: buffer b hi at 2b, lo at 2b + 1
  const uint32_t stages = base + 4 * SN_PLANE;      // filter stages (1024-aligned: SN_PLANE is a multiple of 1024)
  const MbarRing<SN_NST> ring{stages + SN_NST * SN_STAGE};
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < 4 * SN_PLANE / 16; i += blockDim.x) reinterpret_cast<uint4*>(base_ptr)[i] = make_uint4(0, 0, 0, 0);
  ring.init(CONSUMER_WARPS);
  proxy_fence();  // the zeroed halo rows are read by wgmma
  __syncthreads();
  const int n = min(*a.n_dev, a.n_max);
  if (warp == PRODUCER_WARP) {
    if (lane == 0) {
      uint32_t it = 0;
      for (int smp = blockIdx.x; smp < n; smp += gridDim.x)
        for (int l = 0; l < a.nlayers; l++) {
          const uint32_t bytes = 2u * (l == 0 ? 64 : 128) * BK * 2;
          for (int tap = 0; tap < 9; tap++, it++) {
            ring.producer_acquire(it, bytes);
            const uint32_t sb = stages + ring.stage(it) * SN_STAGE;
            tma_load_2d(sb, &maps.hi[l], ring.full(it), tap * BK, 0);
            tma_load_2d(sb + SN_STAGE / 2, &maps.lo[l], ring.full(it), tap * BK, 0);
          }
        }
    }
    return;
  }
  const int tid = threadIdx.x;  // 0..255: the two consumer warpgroups
  uint32_t it = 0;
  bool overflow = false;
  for (int smp = blockIdx.x; smp < n; smp += gridDim.x) {
    // encoder planes -> buffer 0 (the same values k_pack_planes writes for the per-layer path)
    for (int i = tid; i < 128 * 64; i += 256) {
      const int p = i >> 6, c = i & 63;
      const int y = p / a.Wp, x = p - y * a.Wp;
      const float v = plane_input(a.planes, a.F, a.HW, smp, c, y * a.W + x, p < a.S && y < a.H && x < a.W, a.act_scale);
      const uint32_t o = (uint32_t)(c >> 3) * (SN_HR * 16) + (uint32_t)(SN_R0 + p) * 16 + (uint32_t)(c & 7) * 2;
      split_hi_lo(v, *reinterpret_cast<__half*>(base_ptr + o), *reinterpret_cast<__half*>(base_ptr + SN_PLANE + o));
    }
    proxy_fence();
    consumer_sync();
    for (int l = 0; l < a.nlayers; l++) {
      if (l == 0) small_layer<64>(a, l, smp, act, stages, ring, it, 0, overflow);
      else small_layer<128>(a, l, smp, act, stages, ring, it, l & 1, overflow);
      proxy_fence();   // this layer's generic smem writes are read by the next layer's wgmma (async proxy)
      consumer_sync(); // and every warp's MMAs on the buffer the next layer overwrites have completed
    }
  }
  if (overflow) atomicOr(a.err, ERR_ACT_OVERFLOW);
}

// dynamic shared memory opt-in of every instantiation this file launches, on the current device (called from the
// allocator, which runs with the engine's device current)
void tower_configure_device() {
  set_conv_attr<256, true>(); set_conv_attr<128, true>(); set_conv_attr<256, false>(); set_conv_attr<128, false>();
  set_conv_attr<64, false>();
  set_conv_attr<256, true, 1>(); set_conv_attr<256, true, 2>(); set_conv_attr<128, true, 1>(); set_conv_attr<128, true, 2>();
  CUDA_CHECK(cudaFuncSetAttribute(k_net_small, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes_small()));
}

struct Layer {
  int cin, n_total, bn;
  bool pair;
  __half *w_hi = nullptr, *w_lo = nullptr;  // [n_total][9*cin]
  float2* aff = nullptr;                    // [HW][n_total] {A', B} in weight-row order
  CUtensorMap mB_hi, mB_lo;
};
struct Impl {
  NetDims d;
  int n_max, ea, guard, S, rows_alloc, num_sms, passes = TC_PASSES, mode3d = 0, tps = 1;
  bool small = false;  // K = 64, (H+1)(W+1) <= 128: the whole tower of a sample in one kernel (k_net_small)
  __half *xin_hi = nullptr, *xin_lo = nullptr;  // [(guard+rows+guard)][64]
  __half *x_hi[2] = {nullptr, nullptr}, *x_lo[2] = {nullptr, nullptr};  // [(guard+rows+guard)][K]
  CUtensorMap mIn_hi, mIn_lo, mX_hi[2], mX_lo[2];
  std::vector<Layer> layers;
  // profiling
  bool profile = false;
  std::vector<cudaEvent_t> ev_pool;
  size_t ev_used = 0;
  std::vector<std::pair<size_t, size_t>> conv_spans, fwd_spans;  // (start event, stop event)
  size_t ev_get(cudaStream_t st) {
    if (ev_used == ev_pool.size()) { cudaEvent_t e; CUDA_CHECK(cudaEventCreate(&e)); ev_pool.push_back(e); }
    CUDA_CHECK(cudaEventRecord(ev_pool[ev_used], st));
    return ev_used++;
  }
};

// AZ_TC_PASSES (diagnostics) selects 1 or 2 passes for the fused layers; the other shapes always run three
template <int BN>
void launch_fused(int passes, const CUtensorMap& ah, const CUtensorMap& al, const Layer& L, const ConvArgs& a, int num_sms,
                  cudaStream_t st) {
  if (passes == 1) launch_conv<BN, true, 1>(ah, al, L.mB_hi, L.mB_lo, a, num_sms, st);
  else if (passes == 2) launch_conv<BN, true, 2>(ah, al, L.mB_hi, L.mB_lo, a, num_sms, st);
  else launch_conv<BN, true>(ah, al, L.mB_hi, L.mB_lo, a, num_sms, st);
}
void dispatch_conv(const Impl& I, const Layer& L, const CUtensorMap& ah, const CUtensorMap& al, __half* ohi, __half* olo,
                   const int* n_dev, int* err, cudaStream_t st) {
  ConvArgs a;
  a.n_dev = n_dev; a.n_max = I.n_max; a.S = I.S; a.Wp = I.d.W + 1; a.H = I.d.H; a.W = I.d.W; a.guard = I.guard;
  a.mode3d = I.mode3d; a.tps = I.tps;
  a.cin = L.cin; a.n_total = L.n_total; a.cout = I.d.K; a.aff = L.aff; a.out_hi = ohi; a.out_lo = olo;
  a.act_scale = ldexpf(1.0f, I.ea); a.err = err;
  a.out_raw = nullptr; a.exp_a = nullptr; a.exp_b = nullptr;
  if (L.pair && L.bn == 256) launch_fused<256>(I.passes, ah, al, L, a, I.num_sms, st);
  else if (L.pair && L.bn == 128) launch_fused<128>(I.passes, ah, al, L, a, I.num_sms, st);
  else if (!L.pair && L.bn == 256) launch_conv<256, false>(ah, al, L.mB_hi, L.mB_lo, a, I.num_sms, st);
  else if (!L.pair && L.bn == 128) launch_conv<128, false>(ah, al, L.mB_hi, L.mB_lo, a, I.num_sms, st);
  else if (!L.pair && L.bn == 64) launch_conv<64, false>(ah, al, L.mB_hi, L.mB_lo, a, I.num_sms, st);
  else throw std::runtime_error("tc tower: unsupported tile");
}

}  // namespace


bool tc_tower_supported(const NetDims& d) {
  return (d.K == 64 || d.K == 128 || d.K == 256) && d.F <= 64 && d.SharedLayers >= 0;
}

void tc_tower_alloc(TcTower& t, const NetDims& d, int n_max, int act_scale_log2) {
  tower_configure_device();
  Impl* I = new Impl;
  t.impl = I;
  I->d = d; I->n_max = n_max; I->ea = act_scale_log2;
  if (const char* ps = getenv("AZ_TC_PASSES")) { int v = atoi(ps); if (v >= 1 && v <= 3) I->passes = v; }  // experiments only
  // layout choice by padded-row overhead (rows computed per real board point)
  const int S_flat = (d.H + 1) * (d.W + 1), S_ps = d.H * (d.W + 1), tps = (S_ps + BM - 1) / BM;
  I->mode3d = (tps * BM < S_flat) ? 1 : 0;
  if (I->mode3d) { I->guard = 0; I->S = S_ps; I->tps = tps; I->rows_alloc = n_max * I->S; }
  else { I->guard = ((d.W + 2 + 7) / 8) * 8; I->S = S_flat; I->tps = 1; I->rows_alloc = I->guard + n_max * I->S + I->guard + BM; }
  int dev;
  CUDA_CHECK(cudaGetDevice(&dev));
  CUDA_CHECK(cudaDeviceGetAttribute(&I->num_sms, cudaDevAttrMultiProcessorCount, dev));
  auto alloc_h = [&](size_t n) { __half* p; CUDA_CHECK(cudaMalloc(&p, n * 2)); CUDA_CHECK(cudaMemset(p, 0, n * 2)); return p; };
  I->xin_hi = alloc_h((size_t)I->rows_alloc * 64); I->xin_lo = alloc_h((size_t)I->rows_alloc * 64);
  for (int i = 0; i < 2; i++) { I->x_hi[i] = alloc_h((size_t)I->rows_alloc * d.K); I->x_lo[i] = alloc_h((size_t)I->rows_alloc * d.K); }
  if (I->mode3d) {
    I->mIn_hi = make_map3d(I->xin_hi, n_max, I->S, 64); I->mIn_lo = make_map3d(I->xin_lo, n_max, I->S, 64);
    for (int i = 0; i < 2; i++) { I->mX_hi[i] = make_map3d(I->x_hi[i], n_max, I->S, d.K); I->mX_lo[i] = make_map3d(I->x_lo[i], n_max, I->S, d.K); }
  } else {
    I->mIn_hi = make_map(I->xin_hi, I->rows_alloc, 64, BM); I->mIn_lo = make_map(I->xin_lo, I->rows_alloc, 64, BM);
    for (int i = 0; i < 2; i++) { I->mX_hi[i] = make_map(I->x_hi[i], I->rows_alloc, d.K, BM); I->mX_lo[i] = make_map(I->x_lo[i], I->rows_alloc, d.K, BM); }
  }
  // layers: init (single), then SharedLayers fused pairs
  const int K = d.K, HW = d.HW();
  for (int l = 0; l <= d.SharedLayers; l++) {
    Layer L;
    L.pair = l > 0;
    L.cin = l == 0 ? 64 : K;
    L.n_total = L.pair ? 2 * K : K;
    L.bn = std::min(256, L.n_total);
    const size_t ktot = (size_t)9 * L.cin;
    L.w_hi = alloc_h((size_t)L.n_total * ktot); L.w_lo = alloc_h((size_t)L.n_total * ktot);
    CUDA_CHECK(cudaMalloc(&L.aff, (size_t)HW * L.n_total * sizeof(float2)));
    L.mB_hi = make_map(L.w_hi, L.n_total, ktot, L.bn); L.mB_lo = make_map(L.w_lo, L.n_total, ktot, L.bn);
    I->layers.push_back(L);
  }
  I->small = d.K == 64 && !I->mode3d && I->S <= BM && d.W + 2 <= SN_R0 && (int)I->layers.size() <= SN_MAXL && d.F <= 64;
  if (const char* sn = getenv("AZ_TC_SMALLNET")) { if (sn[0] == '0') I->small = false; }  // A/B: the per-layer kernels
  CUDA_CHECK(cudaDeviceSynchronize());
}

int tc_tower_kernel_kind(const TcTower& t) {
  const Impl* I = (const Impl*)t.impl;
  if (!I) return -1;
  return I->small ? 5 : 0;
}

void tc_tower_free(TcTower& t) {
  Impl* I = (Impl*)t.impl;
  if (!I) return;
  cudaFree(I->xin_hi); cudaFree(I->xin_lo);
  for (int i = 0; i < 2; i++) { cudaFree(I->x_hi[i]); cudaFree(I->x_lo[i]); }
  for (Layer& L : I->layers) { cudaFree(L.w_hi); cudaFree(L.w_lo); cudaFree(L.aff); }
  for (cudaEvent_t e : I->ev_pool) cudaEventDestroy(e);
  delete I;
  t.impl = nullptr;
}

// Host-side operand preparation (once per Agent.SwitchToInference): split the fp32 filters into
// fp16 hi/lo at a per-layer power-of-two scale, reorder rows so that an N tile holds the same
// output channels of both branches, fold BN-test (x/sqrt(eps)), gamma and the scales into A'.
void tc_tower_prepare(TcTower& t, const Snapshot& s, cudaStream_t st) {
  Impl* I = (Impl*)t.impl;
  const NetDims& d = I->d;
  const int K = d.K, HW = d.HW();
  CUDA_CHECK(cudaStreamSynchronize(st));
  std::vector<float> h(s.total);
  CUDA_CHECK(cudaMemcpy(h.data(), s.d, s.total * 4, cudaMemcpyDeviceToHost));
  const float inv_sd = 1.0f / sqrtf(1e-5f);
  for (size_t l = 0; l < I->layers.size(); l++) {
    Layer& L = I->layers[l];
    const size_t ktot = (size_t)9 * L.cin;
    const int nb = L.pair ? 2 : 1;
    const SnapUnit* u[2] = {&s.units[l == 0 ? 0 : 1 + 2 * (l - 1)], L.pair ? &s.units[2 + 2 * (l - 1)] : nullptr};
    const int ci_real = u[0]->Ci;
    float mx = 0;
    for (int b = 0; b < nb; b++) {
      const float* f = h.data() + u[b]->filter;
      for (size_t i = 0; i < (size_t)K * ci_real * 9; i++) mx = std::max(mx, std::fabs(f[i]));
    }
    int ew = 0;
    if (mx > 0 && std::isfinite(mx)) { int e2; frexpf(mx, &e2); ew = 7 - e2; }  // mx*2^ew in [64,128)
    const float wscale = ldexpf(1.0f, ew);
    std::vector<__half> whi((size_t)L.n_total * ktot, __float2half_rn(0.0f)), wlo((size_t)L.n_total * ktot, __float2half_rn(0.0f));
    std::vector<float2> aff((size_t)HW * L.n_total);
    const int half_bn = L.pair ? L.bn / 2 : L.bn;
    const float fold = ldexpf(1.0f, -(I->ea + ew)) * inv_sd;
    for (int row = 0; row < L.n_total; row++) {
      const int tile = row / L.bn, q = row % L.bn;
      const int br = L.pair ? (q >= half_bn ? 1 : 0) : 0;
      const int ch = tile * half_bn + (q % half_bn);
      const float* f = h.data() + u[br]->filter + (size_t)ch * ci_real * 9;
      for (int tap = 0; tap < 9; tap++)
        for (int ci = 0; ci < ci_real; ci++) {
          const size_t o = (size_t)row * ktot + (size_t)tap * L.cin + ci;
          split_hi_lo(f[ci * 9 + tap] * wscale, whi[o], wlo[o]);  // filter[co][ci][ky][kx], tap = ky*3+kx
        }
      const float* g = h.data() + u[br]->gamma + (size_t)ch * HW;
      const float* be = h.data() + u[br]->beta + (size_t)ch * HW;
      for (int hw = 0; hw < HW; hw++) aff[(size_t)hw * L.n_total + row] = make_float2(g[hw] * fold, be[hw]);
    }
    CUDA_CHECK(cudaMemcpy(L.w_hi, whi.data(), whi.size() * 2, cudaMemcpyHostToDevice));
    CUDA_CHECK(cudaMemcpy(L.w_lo, wlo.data(), wlo.size() * 2, cudaMemcpyHostToDevice));
    CUDA_CHECK(cudaMemcpy(L.aff, aff.data(), aff.size() * sizeof(float2), cudaMemcpyHostToDevice));
  }
  t.ready = true;
}

void tc_tower_forward(TcTower& t, const NetLayout& NL, const Snapshot& s, Fp32Scratch& sc, const float* planes,
                      const int* n_dev, int n_max, float* policy, int ldp, float* value, int* err_flag, cudaStream_t st,
                      unsigned long long* launches) {
  Impl* I = (Impl*)t.impl;
  if (!I || !t.ready) throw std::runtime_error("tc tower not prepared");
  const NetDims& d = I->d;
  const float scale = ldexpf(1.0f, I->ea);
  const size_t f0 = I->profile ? I->ev_get(st) : 0;
  int cur = 0;
  if (I->small) {  // every conv layer of every leaf in one launch; the head kernels read its output from x_hi[0] / x_lo[0]
    SmallMaps maps;
    SmallNetArgs a;
    a.planes = planes; a.n_dev = n_dev; a.n_max = n_max; a.F = d.F; a.H = d.H; a.W = d.W; a.Wp = d.W + 1; a.S = I->S;
    a.HW = d.HW(); a.nlayers = (int)I->layers.size(); a.guard = I->guard; a.act_scale = scale;
    for (int l = 0; l < SN_MAXL; l++) {
      const Layer& Lr = I->layers[std::min<size_t>(l, I->layers.size() - 1)];
      maps.hi[l] = Lr.mB_hi; maps.lo[l] = Lr.mB_lo; a.aff[l] = Lr.aff;
    }
    a.out_hi = I->x_hi[0]; a.out_lo = I->x_lo[0]; a.err = err_flag;
    const size_t e0 = I->profile ? I->ev_get(st) : 0;
    k_net_small<<<std::max(1, std::min(n_max, I->num_sms)), NTHREADS, smem_bytes_small(), st>>>(maps, a); LAUNCH_CHECK();
    if (I->profile) I->conv_spans.push_back({e0, I->ev_get(st)});
    if (launches) (*launches)++;
  } else {
  {
    size_t total = (size_t)n_max * d.HW() * 64;
    k_pack_planes<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(planes, n_dev, n_max, d.F, d.H, d.W, 64, I->guard, I->S, scale,
                                                                  I->xin_hi, I->xin_lo); LAUNCH_CHECK();
    if (launches) (*launches)++;
  }
  dispatch_conv(*I, I->layers[0], I->mIn_hi, I->mIn_lo, I->x_hi[0], I->x_lo[0], n_dev, err_flag, st);
  if (launches) (*launches)++;
  for (size_t l = 1; l < I->layers.size(); l++) {
    size_t e0 = I->profile ? I->ev_get(st) : 0;
    dispatch_conv(*I, I->layers[l], I->mX_hi[cur], I->mX_lo[cur], I->x_hi[cur ^ 1], I->x_lo[cur ^ 1], n_dev, err_flag, st);
    if (I->profile) I->conv_spans.push_back({e0, I->ev_get(st)});
    if (launches) (*launches)++;
    cur ^= 1;
  }
  }
  {
    const SnapUnit& pu = s.units[1 + 2 * d.SharedLayers];
    const SnapUnit& vu = s.units[2 + 2 * d.SharedLayers];
    size_t warps = (size_t)n_max * d.HW();
    k_head_convs_nhwc<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, st>>>(
        I->x_hi[cur], I->x_lo[cur], n_dev, n_max, d.K, d.H, d.W, I->guard, I->S, 1.0f / scale, s.d + pu.filter, s.d + pu.gamma,
        s.d + pu.beta, s.d + vu.filter, s.d + vu.gamma, s.d + vu.beta, sc.ph, sc.vh); LAUNCH_CHECK();
    if (launches) (*launches)++;
  }
  heads_tiled(NL, s, sc.ph, sc.vh, n_dev, n_max, policy, ldp, value, st, launches);
  if (I->profile) I->fwd_spans.push_back({f0, I->ev_get(st)});
}

void tc_tower_output(TcTower& t, const int* n_dev, int n_max, float* out, cudaStream_t st) {
  const Impl* I = (const Impl*)t.impl;
  if (!I || !t.ready) throw std::runtime_error("tc tower not prepared");
  const NetDims& d = I->d;
  // k_net_small leaves the last layer in buffer 0; the per-layer path swaps buffers once per fused layer
  const int last = I->small ? 0 : (int)(I->layers.size() - 1) & 1;
  const size_t total = (size_t)n_max * d.K * d.HW();
  k_tower_nchw<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(I->x_hi[last], I->x_lo[last], n_dev, n_max, d.K, d.H, d.W, I->guard,
                                                                I->S, ldexpf(1.0f, -I->ea), out); LAUNCH_CHECK();
}

void tc_tower_profile(TcTower& t, bool enable) {
  Impl* I = (Impl*)t.impl;
  if (!I) return;
  I->profile = enable;
  if (enable) { I->ev_used = 0; I->conv_spans.clear(); I->fwd_spans.clear(); }
}
void tc_tower_profile_collect(TcTower& t, cudaStream_t st, double* conv_ms, double* conv_launches, double* fwd_ms,
                              double* fwd_calls) {
  Impl* I = (Impl*)t.impl;
  if (!I) return;
  CUDA_CHECK(cudaStreamSynchronize(st));
  for (auto& sp : I->conv_spans) { float ms; CUDA_CHECK(cudaEventElapsedTime(&ms, I->ev_pool[sp.first], I->ev_pool[sp.second])); *conv_ms += ms; *conv_launches += 1; }
  for (auto& sp : I->fwd_spans) { float ms; CUDA_CHECK(cudaEventElapsedTime(&ms, I->ev_pool[sp.first], I->ev_pool[sp.second])); *fwd_ms += ms; *fwd_calls += 1; }
  I->conv_spans.clear(); I->fwd_spans.clear(); I->ev_used = 0;
}
