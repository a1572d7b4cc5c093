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
//     accumulator; the dropped lo*lo term is ~2^-22 relative.  Under AZ_FLAG_FP16_TOWER the same
//     kernels are instantiated for one fp16 plane per operand (OPS = 1): one pass, no lo buffers;
//   * warp roles (tc_common.cuh): one TMA producer warp, two consumer warpgroups of 64 rows each;
//     smem ring of K-blocks (full/empty mbarriers), persistent CTAs striding over (M-tile, N-tile),
//     epilogue (BN-affine + ReLU + branch add -> fp16 hi/lo split -> global) from the accumulators.
//     The fused layers of K >= 128 nets on hi/lo planes run 192-row tiles (k_conv3x3_m192, three consumer warpgroups):
//     fewer operand bytes per MAC, the same MMA sequence per row; on the per-sample layout the tiles
//     cover the board points alone (TMA im2col), so the zero column and the tile tail cost no MMAs.
// Descriptor bit layouts follow the PTX ISA "Matrix Descriptor Format" table of wgmma.
#include "tc_common.cuh"

namespace {

// the first layer's input at (sample b, channel c, board point hw) before the hi/lo split: the scaled encoder plane, zero
// off the board and in the channels padded beyond F (k_pack_planes and k_net_small write the same operand)
__device__ __forceinline__ float plane_input(const float* planes, int F, int HW, int b, int c, int hw, bool on_board, float scale) {
  return on_board && c < F ? planes[((size_t)b * F + c) * HW + hw] * scale : 0.0f;
}

// a stored activation in fp32: hi + lo, or the single fp16
template <int OPS>
__device__ __forceinline__ float stored_value(const Planes<OPS>& x, size_t o) {
  if constexpr (OPS == 2) return __half2float(x.hi[o]) + __half2float(x.lo[o]);
  else return __half2float(x.hi[o]);
}

// fp32 NCHW planes -> zero-bordered NHWC fp16 hi/lo, or one fp16 (channels padded to cpad)
template <int OPS>
__global__ void k_pack_planes(const float* __restrict__ planes, const int* __restrict__ n_dev, int n_max, int F, int H,
                              int W, int cpad, int guard, int S, float scale, Planes<OPS> out) {
  const int n = min(*n_dev, n_max);
  const int HW = H * W, Wp = W + 1;
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)n * HW * cpad) return;
  const int c = (int)(idx % cpad);
  const int hw = (int)((idx / cpad) % HW);
  const int b = (int)(idx / ((size_t)cpad * HW));
  const int y = hw / W, x = hw - y * W;
  const float v = plane_input(planes, F, HW, b, c, hw, true, scale);
  const size_t o = ((size_t)guard + (size_t)b * S + y * Wp + x) * cpad + c;
  if constexpr (OPS == 2) split_hi_lo(v, out.hi[o], out.lo[o]);
  else out.hi[o] = __float2half_rn(v);
}
// The two 1x1 head convs (K->2 policy, K->1 value; dual.go:70,85) + BN-test affine + ReLU straight
// from the tower's NHWC hi/lo (or single fp16) output: one warp per board point, lanes split the channels
// (coalesced 16-byte loads), three dot products reduced with shuffles.
//   ph [n][2][HW], vh [n][HW]  (the layout the linear layers consume)
template <int OPS>
__global__ void k_head_convs_nhwc(const Planes<OPS> act, const int* __restrict__ n_dev,
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
    const uint4 h4 = *(const uint4*)(act.hi + row * K + c0);
    uint4 l4;
    if constexpr (OPS == 2) l4 = *(const uint4*)(act.lo + row * K + c0);
    const __half* hh = (const __half*)&h4;
    const __half* ll = (const __half*)&l4;
#pragma unroll
    for (int i = 0; i < 8; i++) {
      float v;
      if constexpr (OPS == 2) v = (__half2float(hh[i]) + __half2float(ll[i])) * inv_scale;
      else v = __half2float(hh[i]) * inv_scale;
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
// diagnostics: the NHWC tower output (the values k_head_convs_nhwc reads) -> fp32 NCHW [n][K][HW]
template <int OPS>
__global__ void k_tower_nchw(const Planes<OPS> act, const int* __restrict__ n_dev, int n_max, int K, int H, int W, int guard, int S,
                             float inv_scale, float* out) {
  const int n = min(*n_dev, n_max);
  const int HW = H * W, Wp = W + 1;
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)n * K * HW) return;
  const int hw = (int)(idx % HW), c = (int)((idx / HW) % K), b = (int)(idx / ((size_t)HW * K));
  const int y = hw / W, x = hw - y * W;
  const size_t o = ((size_t)guard + (size_t)b * S + y * Wp + x) * K + c;
  out[idx] = stored_value<OPS>(act, o) * inv_scale;
}

// -------------------------------------------------------------------------------------------------
// k_net_small: the whole tower of a K = 64 net on a board of at most 128 padded positions ((H+1)(W+1) <= 128, BASELINE
// C2) in one persistent kernel.  A 3x3 convolution mixes board points of one sample only, so a CTA carries a sample
// through every layer with no grid-wide step: the sample's zero-bordered positions x 64 channels stay in shared memory as
// fp16 hi / lo planes (two ping-pong buffers), only the filters stream from L2 (TMA into an mbarrier ring that runs ahead
// across layers and samples, one stage per (layer, tap)), and the last layer writes the NHWC hi/lo buffer the head
// kernels read.  Activations are stored K-major without swizzle ([8-channel chunk][row][16 B]), so tap (dy, dx) is the
// same tile with its descriptor starting dy*(W+1)+dx rows further — no copy per tap.  Same MMA sequence (tap by tap, three
// passes), same epilogue arithmetic as the per-layer kernels: the outputs are identical to that path.  The body is
// instantiated for both operand forms: k_net_small (hi/lo planes, three passes) and k_smallnet_fp16 (one fp16 plane per
// operand, one pass, the epilogue of k_conv3x3_tc's single-plane form); the freed shared memory deepens the filter ring.
constexpr int SN_MAXL = 8;                 // init conv + up to 7 blocks
constexpr int SN_R0 = 16;                  // halo rows in front of the tile (>= W + 2)
constexpr int SN_HR = 160;                 // rows per activation plane: halo + 128 + halo
constexpr int SN_PLANE = 8 * SN_HR * 16;   // one fp16 plane: 8 chunks of 8 channels x SN_HR rows x 16 B
constexpr int SN_TILE = 128 * BK * 2;      // one filter plane of up to 128 rows x 64 K
// a filter stage holds OPS planes; the ring takes what the two activation buffers leave (4 stages for hi/lo, 11 for fp16)
__host__ __device__ constexpr int sn_stage_bytes(int OPS) { return OPS * SN_TILE; }
__host__ __device__ constexpr int sn_stages(int OPS) { return (SMEM_RING_BUDGET - 2 * OPS * SN_PLANE) / sn_stage_bytes(OPS); }
__host__ __device__ constexpr int smem_bytes_small(int OPS) {
  return 2 * OPS * SN_PLANE + sn_stages(OPS) * sn_stage_bytes(OPS) + 1024 + 256;
}
template <int OPS> struct SmallMaps { PlaneMaps<OPS> w[SN_MAXL]; };
template <int OPS>
struct SmallNetArgs {
  const float* planes;  // [n][F][HW] encoder planes
  const int* n_dev;
  int n_max, F, H, W, Wp, S, HW, nlayers, guard;
  float act_scale;
  const float2* aff[SN_MAXL];  // per layer [HW][n_total] {A', B}
  Planes<OPS> out;             // last layer: [(guard + n*S)][64], the layout k_head_convs_nhwc reads
  int* err;
};

// one layer of one sample: 9 taps of the filter ring into acc, then the epilogue into smem (or global for the last layer)
template <int N, int OPS>
__device__ __forceinline__ void small_layer(const SmallNetArgs<OPS>& a, int l, int smp, uint32_t act, uint32_t stages,
                                            const MbarRing<sn_stages(OPS)>& ring, uint32_t& it, int in, bool& overflow) {
  constexpr bool PAIR = N == 128;
  constexpr int OUTC = PAIR ? N / 2 : N;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
  int row0, col0;
  acc_frag_origin(warp, lane, row0, col0);
  const uint32_t in_hi = act + (OPS * in) * SN_PLANE;
  float acc[N / 2];
  for (int tap = 0; tap < 9; tap++, it++) {
    ring.consumer_wait(it);
    const uint32_t shift = (uint32_t)(SN_R0 + wg * 64 + (tap / 3 - 1) * a.Wp + (tap % 3 - 1)) * 16;
    const uint32_t sb = stages + ring.stage(it) * sn_stage_bytes(OPS);
    mma_kblock<N, 0, OPS>(acc, make_desc_plain(in_hi + shift, SN_HR * 16), make_desc_plain(in_hi + SN_PLANE + shift, SN_HR * 16),
                          make_desc_sw(sb), make_desc_sw(sb + SN_TILE), 32 >> 4, tap == 0, 2 * SN_HR * 16 >> 4);
    ring.consumer_release(it);
  }
  const bool last = l == a.nlayers - 1;
  const uint32_t out_hi = act + (OPS * (in ^ 1)) * SN_PLANE;
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
        const float v = valid ? fused_value<N, PAIR>(aff, acc, j, h, e, a.act_scale) : 0.0f;
        if constexpr (OPS == 2) split_hi_lo(v, hv[e], lv[e]);
        else hv[e] = __float2half_rn(v);
        overflow |= !(fabsf(__half2float(hv[e])) <= 65504.0f);
      }
      const int c = 8 * j + col0;
      if (last) {
        *reinterpret_cast<__half2*>(a.out.hi + grow * 64 + c) = __halves2half2(hv[0], hv[1]);
        if constexpr (OPS == 2) *reinterpret_cast<__half2*>(a.out.lo + grow * 64 + c) = __halves2half2(lv[0], lv[1]);
      } else {  // chunk c / 8, row SN_R0 + p, byte (c % 8) * 2; invalid positions are written as zeros
        const uint32_t o = (uint32_t)(c >> 3) * (SN_HR * 16) + (uint32_t)(SN_R0 + p) * 16 + (uint32_t)(c & 7) * 2;
        const __half2 h2 = __halves2half2(hv[0], hv[1]);
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(out_hi + o), "r"(*reinterpret_cast<const uint32_t*>(&h2)) : "memory");
        if constexpr (OPS == 2) {
          const __half2 l2 = __halves2half2(lv[0], lv[1]);
          asm volatile("st.shared.b32 [%0], %1;" ::"r"(out_hi + SN_PLANE + o), "r"(*reinterpret_cast<const uint32_t*>(&l2)) : "memory");
        }
      }
    }
  }
}

__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }
__device__ __forceinline__ void proxy_fence() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

template <int OPS>
__device__ __forceinline__ void net_small(const SmallMaps<OPS>& maps, const SmallNetArgs<OPS>& a) {
  constexpr int NST = sn_stages(OPS);
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* base_ptr = smem_raw + (base - smem_u32(smem_raw));
  const uint32_t act = base;                         // 2 * OPS planes: buffer b hi at OPS*b, lo (OPS = 2) at 2b + 1
  const uint32_t stages = base + 2 * OPS * SN_PLANE;  // filter stages (1024-aligned: SN_PLANE is a multiple of 1024)
  const MbarRing<NST> ring{stages + NST * sn_stage_bytes(OPS)};
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < 2 * OPS * SN_PLANE / 16; i += blockDim.x) reinterpret_cast<uint4*>(base_ptr)[i] = make_uint4(0, 0, 0, 0);
  ring.init(CONSUMER_WARPS);
  proxy_fence();  // the zeroed halo rows are read by wgmma
  __syncthreads();
  const int n = min(*a.n_dev, a.n_max);
  if (warp == PRODUCER_WARP) {
    if (lane == 0) {
      uint32_t it = 0;
      for (int smp = blockIdx.x; smp < n; smp += gridDim.x)
        for (int l = 0; l < a.nlayers; l++) {
          const uint32_t bytes = OPS * (l == 0 ? 64 : 128) * BK * 2;
          for (int tap = 0; tap < 9; tap++, it++) {
            ring.producer_acquire(it, bytes);
            const uint32_t sb = stages + ring.stage(it) * sn_stage_bytes(OPS);
            tma_load_2d(sb, &maps.w[l].hi, ring.full(it), tap * BK, 0);
            if constexpr (OPS == 2) tma_load_2d(sb + SN_TILE, &maps.w[l].lo, ring.full(it), tap * BK, 0);
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
      if constexpr (OPS == 2) split_hi_lo(v, *reinterpret_cast<__half*>(base_ptr + o), *reinterpret_cast<__half*>(base_ptr + SN_PLANE + o));
      else *reinterpret_cast<__half*>(base_ptr + o) = __float2half_rn(v);
    }
    proxy_fence();
    consumer_sync();
    for (int l = 0; l < a.nlayers; l++) {
      if (l == 0) small_layer<64, OPS>(a, l, smp, act, stages, ring, it, 0, overflow);
      else small_layer<128, OPS>(a, l, smp, act, stages, ring, it, l & 1, overflow);
      proxy_fence();   // this layer's generic smem writes are read by the next layer's wgmma (async proxy)
      consumer_sync(); // and every warp's MMAs on the buffer the next layer overwrites have completed
    }
  }
  if (overflow) atomicOr(a.err, ERR_ACT_OVERFLOW);
}
__global__ void __launch_bounds__(NTHREADS, 1) k_net_small(const __grid_constant__ SmallMaps<2> maps, SmallNetArgs<2> a) {
  net_small<2>(maps, a);
}
__global__ void __launch_bounds__(NTHREADS, 1) k_smallnet_fp16(const __grid_constant__ SmallMaps<1> maps, SmallNetArgs<1> a) {
  net_small<1>(maps, a);
}

// dynamic shared memory opt-in of every instantiation this file launches, on the current device (called from the
// allocator, which runs with the engine's device current)
void tower_configure_device() {
  set_conv_attr<3, 256, true>();
  set_conv_attr<2, 256, true>(); set_conv_attr<2, 128, true>(); set_conv_attr<2, 256, false>(); set_conv_attr<2, 128, false>();
  set_conv_attr<2, 64, false>();
  set_conv_attr<2, 256, true, 1>(); set_conv_attr<2, 128, true, 1>(); set_conv_attr<2, 256, false, 1>();
  set_conv_attr<2, 128, false, 1>(); set_conv_attr<2, 64, false, 1>();
  CUDA_CHECK(cudaFuncSetAttribute(k_net_small, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes_small(2)));
  CUDA_CHECK(cudaFuncSetAttribute(k_smallnet_fp16, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes_small(1)));
}

struct Layer {
  int cin, n_total, bn;
  bool pair;
  __half *w_hi = nullptr, *w_lo = nullptr;  // [n_total][9*cin]; no w_lo in fp16 mode
  float2* aff = nullptr;                    // [HW][n_total] {A', B} in weight-row order
  CUtensorMap mB_hi, mB_lo;
};
struct Impl {
  NetDims d;
  int n_max, ea, guard, S, rows_alloc, num_sms, mode3d = 0, tps = 1;
  bool fp16 = false;   // AZ_FLAG_FP16_TOWER: one fp16 plane per operand (no *_lo buffers or maps), one pass
  bool small = false;  // K = 64, (H+1)(W+1) <= 128: the whole tower of a sample in one kernel (k_net_small / k_smallnet_fp16)
  bool m192 = false;   // the fused layers run k_conv3x3_m192 (192-row tiles)
  __half *xin_hi = nullptr, *xin_lo = nullptr;  // [(guard+rows+guard)][64]
  __half *x_hi[2] = {nullptr, nullptr}, *x_lo[2] = {nullptr, nullptr};  // [(guard+rows+guard)][K]
  CUtensorMap mIn_hi, mIn_lo, mX_hi[2], mX_lo[2];
  CUtensorMap mX192_hi[2], mX192_lo[2];  // the same buffers with 192-row boxes (m192 only)
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

// the host's view of one operand in the kernels' form: hi and lo, or hi alone (lo is not allocated in fp16 mode)
template <int OPS> Planes<OPS> planes_of(__half* hi, __half* lo) {
  if constexpr (OPS == 2) return {hi, lo};
  else return {hi};
}
template <int OPS> PlaneMaps<OPS> maps_of(const CUtensorMap& hi, const CUtensorMap& lo) {
  if constexpr (OPS == 2) return {hi, lo};
  else return {hi};
}

// A192: the input's 192-row maps when the fused layers run k_conv3x3_m192 (I.m192), else nullptr
template <int OPS>
void dispatch_conv(const Impl& I, const Layer& L, const PlaneMaps<OPS>& A, const PlaneMaps<OPS>* A192, const Planes<OPS>& out,
                   const int* n_dev, int* err, cudaStream_t st) {
  ConvArgs a;
  a.n_dev = n_dev; a.n_max = I.n_max; a.S = I.S; a.Wp = I.d.W + 1; a.H = I.d.H; a.W = I.d.W; a.guard = I.guard;
  a.mode3d = I.mode3d; a.tps = I.tps;
  a.cin = L.cin; a.n_total = L.n_total; a.cout = I.d.K; a.aff = L.aff;
  a.act_scale = ldexpf(1.0f, I.ea); a.err = err;
  a.out_raw = nullptr; a.exp_a = nullptr; a.exp_b = nullptr;
  const PlaneMaps<OPS> B = maps_of<OPS>(L.mB_hi, L.mB_lo);
  if constexpr (OPS == 2)  // the 192-row kernel exists for hi/lo planes only
    if (A192 && L.pair && L.bn == 256) return launch_conv<3, 256, true>(*A192, B, a, out, I.num_sms, st);
  if (L.pair && L.bn == 256) launch_conv<2, 256, true, OPS>(A, B, a, out, I.num_sms, st);
  else if (L.pair && L.bn == 128) launch_conv<2, 128, true, OPS>(A, B, a, out, I.num_sms, st);
  else if (!L.pair && L.bn == 256) launch_conv<2, 256, false, OPS>(A, B, a, out, I.num_sms, st);
  else if (!L.pair && L.bn == 128) launch_conv<2, 128, false, OPS>(A, B, a, out, I.num_sms, st);
  else if (!L.pair && L.bn == 64) launch_conv<2, 64, false, OPS>(A, B, a, out, I.num_sms, st);
  else throw std::runtime_error("tc tower: unsupported tile");
}

}  // namespace


bool tc_tower_supported(const NetDims& d) {
  return (d.K == 64 || d.K == 128 || d.K == 256) && d.F <= 64 && d.SharedLayers >= 0;
}

void tc_tower_alloc(TcTower& t, const NetDims& d, int n_max, int act_scale_log2, bool fp16) {
  tower_configure_device();
  Impl* I = new Impl;
  t.impl = I;
  I->d = d; I->n_max = n_max; I->ea = act_scale_log2; I->fp16 = fp16;
  // layout choice by padded-row overhead (rows computed per real board point)
  const int S_flat = (d.H + 1) * (d.W + 1), S_ps = d.H * (d.W + 1), tps = (S_ps + BM - 1) / BM;
  I->mode3d = (tps * BM < S_flat) ? 1 : 0;
  if (I->mode3d) { I->guard = 0; I->S = S_ps; I->tps = tps; I->rows_alloc = n_max * I->S; }
  else { I->guard = ((d.W + 2 + 7) / 8) * 8; I->S = S_flat; I->tps = 1; I->rows_alloc = I->guard + n_max * I->S + I->guard + BM; }
  int dev;
  CUDA_CHECK(cudaGetDevice(&dev));
  CUDA_CHECK(cudaDeviceGetAttribute(&I->num_sms, cudaDevAttrMultiProcessorCount, dev));
  auto alloc_h = [&](size_t n) { __half* p; CUDA_CHECK(cudaMalloc(&p, n * 2)); CUDA_CHECK(cudaMemset(p, 0, n * 2)); return p; };
  // an activation buffer [(guard+rows+guard)][cols] and its tensor map; the lo planes exist only in the hi/lo form
  auto act_buf = [&](int cols, __half*& p, CUtensorMap& m) {
    p = alloc_h((size_t)I->rows_alloc * cols);
    m = I->mode3d ? make_map3d(p, n_max, I->S, cols) : make_map(p, I->rows_alloc, cols, BM);
  };
  act_buf(64, I->xin_hi, I->mIn_hi);
  if (!fp16) act_buf(64, I->xin_lo, I->mIn_lo);
  for (int i = 0; i < 2; i++) {
    act_buf(d.K, I->x_hi[i], I->mX_hi[i]);
    if (!fp16) act_buf(d.K, I->x_lo[i], I->mX_lo[i]);
  }
  // 192-row tiles for the fused layers (BN = 256: K >= 128) of the three-pass hi/lo tower.  On the per-sample layout
  // their rows are the n * H * W board points alone, gathered by im2col maps (19x19: 361 rows per sample against 384 of
  // the 128-row tiles); on the flat layout they are the flat rows, padded at the batch end only.  The storage layout
  // above stays the 128-row one; TMA zero-fills what a box reads past it or off the board.
  I->m192 = !fp16 && d.K >= 128;
  if (const char* m = getenv("AZ_TC_M192")) { if (m[0] == '0') I->m192 = false; }  // A/B: the 128-row kernel
  if (I->m192)
    for (int i = 0; i < 2; i++) {
      __half* p[2] = {I->x_hi[i], I->x_lo[i]};
      CUtensorMap* m[2] = {&I->mX192_hi[i], &I->mX192_lo[i]};
      for (int j = 0; j < 2; j++)
        *m[j] = I->mode3d ? make_map_im2col(p[j], n_max, d.H, d.W, d.K, BM192) : make_map(p[j], I->rows_alloc, d.K, BM192);
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
    L.w_hi = alloc_h((size_t)L.n_total * ktot);
    L.mB_hi = make_map(L.w_hi, L.n_total, ktot, L.bn);
    if (!fp16) { L.w_lo = alloc_h((size_t)L.n_total * ktot); L.mB_lo = make_map(L.w_lo, L.n_total, ktot, L.bn); }
    CUDA_CHECK(cudaMalloc(&L.aff, (size_t)HW * L.n_total * sizeof(float2)));
    I->layers.push_back(L);
  }
  I->small = d.K == 64 && !I->mode3d && I->S <= BM && d.W + 2 <= SN_R0 && (int)I->layers.size() <= SN_MAXL && d.F <= 64;
  if (const char* sn = getenv("AZ_TC_SMALLNET")) { if (sn[0] == '0') I->small = false; }  // A/B: the per-layer kernels
  CUDA_CHECK(cudaDeviceSynchronize());
}

int tc_tower_kernel_kind(const TcTower& t) {
  const Impl* I = (const Impl*)t.impl;
  if (!I) return -1;
  if (I->fp16) return I->small ? 7 : 6;
  return I->small ? 5 : I->m192 ? 8 : 0;
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
// fp16 hi/lo (fp16 mode: round them to one fp16) at a per-layer power-of-two scale, reorder rows so that an N tile holds the same
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
    std::vector<__half> whi((size_t)L.n_total * ktot, __float2half_rn(0.0f)), wlo(I->fp16 ? 0 : whi.size(), __float2half_rn(0.0f));
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
          const float w = f[ci * 9 + tap] * wscale;  // filter[co][ci][ky][kx], tap = ky*3+kx
          if (I->fp16) whi[o] = __float2half_rn(w);
          else split_hi_lo(w, whi[o], wlo[o]);
        }
      const float* g = h.data() + u[br]->gamma + (size_t)ch * HW;
      const float* be = h.data() + u[br]->beta + (size_t)ch * HW;
      for (int hw = 0; hw < HW; hw++) aff[(size_t)hw * L.n_total + row] = make_float2(g[hw] * fold, be[hw]);
    }
    CUDA_CHECK(cudaMemcpy(L.w_hi, whi.data(), whi.size() * 2, cudaMemcpyHostToDevice));
    if (!I->fp16) CUDA_CHECK(cudaMemcpy(L.w_lo, wlo.data(), wlo.size() * 2, cudaMemcpyHostToDevice));
    CUDA_CHECK(cudaMemcpy(L.aff, aff.data(), aff.size() * sizeof(float2), cudaMemcpyHostToDevice));
  }
  t.ready = true;
}

template <int OPS>
void tower_forward(Impl* I, const NetLayout& NL, const Snapshot& s, Fp32Scratch& sc, const float* planes, const int* n_dev,
                   int n_max, float* policy, int ldp, float* value, int* err_flag, cudaStream_t st, unsigned long long* launches) {
  const NetDims& d = I->d;
  const float scale = ldexpf(1.0f, I->ea);
  const size_t f0 = I->profile ? I->ev_get(st) : 0;
  int cur = 0;
  if (I->small) {  // every conv layer of every leaf in one launch; the head kernels read its output from buffer 0
    SmallMaps<OPS> maps;
    SmallNetArgs<OPS> a;
    a.planes = planes; a.n_dev = n_dev; a.n_max = n_max; a.F = d.F; a.H = d.H; a.W = d.W; a.Wp = d.W + 1; a.S = I->S;
    a.HW = d.HW(); a.nlayers = (int)I->layers.size(); a.guard = I->guard; a.act_scale = scale;
    for (int l = 0; l < SN_MAXL; l++) {
      const Layer& Lr = I->layers[std::min<size_t>(l, I->layers.size() - 1)];
      maps.w[l] = maps_of<OPS>(Lr.mB_hi, Lr.mB_lo); a.aff[l] = Lr.aff;
    }
    a.out = planes_of<OPS>(I->x_hi[0], I->x_lo[0]); a.err = err_flag;
    const size_t e0 = I->profile ? I->ev_get(st) : 0;
    const int grid = std::max(1, std::min(n_max, I->num_sms));
    if constexpr (OPS == 2) k_net_small<<<grid, NTHREADS, smem_bytes_small(OPS), st>>>(maps, a);
    else k_smallnet_fp16<<<grid, NTHREADS, smem_bytes_small(OPS), st>>>(maps, a);
    LAUNCH_CHECK();
    if (I->profile) I->conv_spans.push_back({e0, I->ev_get(st)});
    if (launches) (*launches)++;
  } else {
  {
    size_t total = (size_t)n_max * d.HW() * 64;
    k_pack_planes<OPS><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(planes, n_dev, n_max, d.F, d.H, d.W, 64, I->guard, I->S,
                                                                       scale, planes_of<OPS>(I->xin_hi, I->xin_lo)); LAUNCH_CHECK();
    if (launches) (*launches)++;
  }
  dispatch_conv<OPS>(*I, I->layers[0], maps_of<OPS>(I->mIn_hi, I->mIn_lo), nullptr, planes_of<OPS>(I->x_hi[0], I->x_lo[0]), n_dev,
                     err_flag, st);
  if (launches) (*launches)++;
  for (size_t l = 1; l < I->layers.size(); l++) {
    size_t e0 = I->profile ? I->ev_get(st) : 0;
    const PlaneMaps<OPS> A192 = maps_of<OPS>(I->mX192_hi[cur], I->mX192_lo[cur]);
    dispatch_conv<OPS>(*I, I->layers[l], maps_of<OPS>(I->mX_hi[cur], I->mX_lo[cur]), I->m192 ? &A192 : nullptr,
                       planes_of<OPS>(I->x_hi[cur ^ 1], I->x_lo[cur ^ 1]), n_dev, err_flag, st);
    if (I->profile) I->conv_spans.push_back({e0, I->ev_get(st)});
    if (launches) (*launches)++;
    cur ^= 1;
  }
  }
  {
    const SnapUnit& pu = s.units[1 + 2 * d.SharedLayers];
    const SnapUnit& vu = s.units[2 + 2 * d.SharedLayers];
    size_t warps = (size_t)n_max * d.HW();
    k_head_convs_nhwc<OPS><<<(unsigned)((warps * 32 + 255) / 256), 256, 0, st>>>(
        planes_of<OPS>(I->x_hi[cur], I->x_lo[cur]), n_dev, n_max, d.K, d.H, d.W, I->guard, I->S, 1.0f / scale, s.d + pu.filter,
        s.d + pu.gamma, s.d + pu.beta, s.d + vu.filter, s.d + vu.gamma, s.d + vu.beta, sc.ph, sc.vh); LAUNCH_CHECK();
    if (launches) (*launches)++;
  }
  heads_tiled(NL, s, sc.ph, sc.vh, n_dev, n_max, policy, ldp, value, st, launches);
  if (I->profile) I->fwd_spans.push_back({f0, I->ev_get(st)});
}

void tc_tower_forward(TcTower& t, const NetLayout& NL, const Snapshot& s, Fp32Scratch& sc, const float* planes,
                      const int* n_dev, int n_max, float* policy, int ldp, float* value, int* err_flag, cudaStream_t st,
                      unsigned long long* launches) {
  Impl* I = (Impl*)t.impl;
  if (!I || !t.ready) throw std::runtime_error("tc tower not prepared");
  if (I->fp16) tower_forward<1>(I, NL, s, sc, planes, n_dev, n_max, policy, ldp, value, err_flag, st, launches);
  else tower_forward<2>(I, NL, s, sc, planes, n_dev, n_max, policy, ldp, value, err_flag, st, launches);
}

void tc_tower_output(TcTower& t, const int* n_dev, int n_max, float* out, cudaStream_t st) {
  const Impl* I = (const Impl*)t.impl;
  if (!I || !t.ready) throw std::runtime_error("tc tower not prepared");
  const NetDims& d = I->d;
  // k_net_small leaves the last layer in buffer 0; the per-layer path swaps buffers once per fused layer
  const int last = I->small ? 0 : (int)(I->layers.size() - 1) & 1;
  const size_t total = (size_t)n_max * d.K * d.HW();
  const unsigned blocks = (unsigned)((total + 255) / 256);
  const float inv_scale = ldexpf(1.0f, -I->ea);
  if (I->fp16)
    k_tower_nchw<1><<<blocks, 256, 0, st>>>(planes_of<1>(I->x_hi[last], nullptr), n_dev, n_max, d.K, d.H, d.W, I->guard, I->S,
                                            inv_scale, out);
  else
    k_tower_nchw<2><<<blocks, 256, 0, st>>>(planes_of<2>(I->x_hi[last], I->x_lo[last]), n_dev, n_max, d.K, d.H, d.W, I->guard, I->S,
                                            inv_scale, out);
  LAUNCH_CHECK();
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
