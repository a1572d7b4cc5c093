// agogo_b200 — dual network parameter layout, init, inference snapshot and the fp32 CUDA-core
// forward.  The fp32 forward is the validation-grade path (and the production path for nets too
// small for tensor cores: tic-tac-toe K=3, Connect-4 K=16): one thread per output element, taps
// accumulated in ascending (ci, ky, kx) order with unfused multiply and add, i.e. the same
// rounding sequence as the oracle's restatement (dualnet/ermahagerdmonards.go:33-73).
// Compiled with -fmad=false.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdio>
#include <stdexcept>
#include <thread>

#include "nn.cuh"

// ---------------------------------------------------------------------------------------------
// layout: dual.Model() = graph-creation order (dual.go:50-103, 134-142)
static int add_param(NetLayout& L, const std::string& name, std::vector<int> shape, int init) {
  ParamDescH d;
  d.name = name; d.rank = (int)shape.size(); d.init = init;
  size_t sz = 1;
  for (int i = 0; i < 4; i++) { d.shape[i] = i < d.rank ? shape[i] : 1; if (i < d.rank) sz *= shape[i]; }
  d.offset = L.total; d.size = sz;
  L.total += sz;
  L.desc.push_back(d);
  return (int)L.desc.size() - 1;
}
static void add_unit(NetLayout& L, const std::string& name, int Ci, int Co, int k) {
  UnitH u;
  u.Ci = Ci; u.Co = Co; u.k = k;
  u.filter = add_param(L, "Filter" + name, {Co, Ci, k, k}, 1);                      // GlorotU(1.0), ermahagerdmonards.go:39
  u.gamma = add_param(L, "Filter" + name + "_conv_γ", {L.d.B, Co, L.d.H, L.d.W}, 2);  // created by BatchNorm(x,nil,nil)
  u.beta = add_param(L, "Filter" + name + "_conv_β", {L.d.B, Co, L.d.H, L.d.W}, 2);
  L.units.push_back(u);
}
NetLayout build_layout(const NetDims& d) {
  NetLayout L;
  L.d = d;
  const int HW = d.HW();
  add_unit(L, "Init", d.F, d.K, 3);
  for (int i = 0; i < d.SharedLayers; i++) {
    char buf[64];
    snprintf(buf, sizeof buf, "Layer1 of Shared Layer %d", i); add_unit(L, buf, d.K, d.K, 3);
    snprintf(buf, sizeof buf, "Layer2 of Shared Layer %d", i); add_unit(L, buf, d.K, d.K, 3);
  }
  add_unit(L, "PolicyHead", d.K, 2, 1);
  L.pW = add_param(L, "Policy_w", {2 * HW, d.A1}, 2);  // GlorotN(1.0), ermahagerdmonards.go:80
  L.pB = add_param(L, "Policy_b", {d.B, d.A1}, 0);     // shaped like xw (batch-shaped), zeros
  add_unit(L, "ValueHead", d.K, 1, 1);
  L.vW = add_param(L, "Value_w", {HW, d.FC}, 2);
  L.vB = add_param(L, "Value_b", {d.B, d.FC}, 0);
  L.voW = add_param(L, "ValueOutput_w", {d.FC, 1}, 2);
  L.voB = add_param(L, "ValueOutput_b", {d.B, 1}, 0);
  return L;
}

// injected RNG: same specification as the oracle (splitmix64; see DESIGN.md "determinism")
static inline uint64_t splitmix64(uint64_t* s) {
  uint64_t z = (*s += 0x9E3779B97F4A7C15ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
static inline uint64_t derive_seed(uint64_t seed, uint64_t stream) {
  uint64_t s = seed ^ (0xD1B54A32D192ED03ull * (stream + 1));
  return splitmix64(&s);
}
// splitmix64 is counter based (state_i = s0 + i*GOLDEN), so every tensor's stream can be generated
// in independent chunks on many host threads and still be bit-identical to the sequential draw.
static inline uint64_t splitmix_at(uint64_t s0, uint64_t i) {
  uint64_t z = s0 + (i + 1) * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
void init_params_host(const NetLayout& L, uint64_t seed, std::vector<float>* out) {
  out->assign(L.total, 0.0f);
  struct Job { size_t t, lo, hi; };
  std::vector<Job> jobs;
  const size_t CH = 1 << 20;
  for (size_t t = 0; t < L.desc.size(); t++)
    if (L.desc[t].init) for (size_t lo = 0; lo < L.desc[t].size; lo += CH) jobs.push_back({t, lo, std::min(L.desc[t].size, lo + CH)});
  std::atomic<size_t> next{0};
  auto work = [&]() {
    for (;;) {
      size_t j = next.fetch_add(1);
      if (j >= jobs.size()) return;
      const ParamDescH& d = L.desc[jobs[j].t];
      float* p = out->data() + d.offset;
      double field = 1;
      for (int i = 2; i < d.rank; i++) field *= d.shape[i];
      const double fan = (double)(d.shape[0] + d.shape[1]) * field;
      const double stdev = 1.0 * std::sqrt(2.0 / fan);
      const uint64_t s0 = derive_seed(seed, jobs[j].t);
      if (d.init == 1) {
        const float lim = (float)(stdev * std::sqrt(3.0));
        for (size_t i = jobs[j].lo; i < jobs[j].hi; i++) {
          float u = (float)(splitmix_at(s0, i) >> 40) * (1.0f / 16777216.0f);
          p[i] = (2.0f * u - 1.0f) * lim;
        }
      } else {
        const float sd = (float)stdev;
        for (size_t i = jobs[j].lo; i < jobs[j].hi; i++) {
          double u1 = ((double)(splitmix_at(s0, 2 * i) >> 11) + 1.0) * (1.0 / 9007199254740992.0);
          double u2 = ((double)(splitmix_at(s0, 2 * i + 1) >> 11)) * (1.0 / 9007199254740992.0);
          float nrm = (float)(std::sqrt(-2.0 * std::log(u1)) * std::cos(6.283185307179586476925 * u2));
          p[i] = nrm * sd;
        }
      }
    }
  };
  unsigned nt = std::max(1u, std::min(64u, std::thread::hardware_concurrency()));
  if (jobs.size() < 4) nt = 1;
  std::vector<std::thread> th;
  for (unsigned i = 1; i < nt; i++) th.emplace_back(work);
  work();
  for (auto& t : th) t.join();
}

// ---------------------------------------------------------------------------------------------
Snapshot make_snapshot_layout(const NetLayout& L) {
  Snapshot s;
  size_t off = 0;
  const int HW = L.d.HW();
  for (const UnitH& u : L.units) {
    SnapUnit su;
    su.Ci = u.Ci; su.Co = u.Co; su.k = u.k;
    su.filter = off; off += (size_t)u.Co * u.Ci * u.k * u.k;
    su.gamma = off; off += (size_t)u.Co * HW;
    su.beta = off; off += (size_t)u.Co * HW;
    s.units.push_back(su);
  }
  s.pW = off; off += (size_t)2 * HW * L.d.A1;
  s.pB = off; off += L.d.A1;
  s.vW = off; off += (size_t)HW * L.d.FC;
  s.vB = off; off += L.d.FC;
  s.voW = off; off += L.d.FC;
  s.voB = off; off += 1;
  s.total = off;
  return s;
}
void snapshot_gather(const NetLayout& L, const float* p, Snapshot& s, cudaStream_t st) {
  const int HW = L.d.HW();
  auto cp = [&](size_t dst, size_t src, size_t n) {
    CUDA_CHECK(cudaMemcpyAsync(s.d + dst, p + src, n * 4, cudaMemcpyDeviceToDevice, st));
  };
  for (size_t i = 0; i < L.units.size(); i++) {
    const UnitH& u = L.units[i];
    cp(s.units[i].filter, L.desc[u.filter].offset, L.desc[u.filter].size);
    cp(s.units[i].gamma, L.desc[u.gamma].offset, (size_t)u.Co * HW);  // batch row 0
    cp(s.units[i].beta, L.desc[u.beta].offset, (size_t)u.Co * HW);
  }
  cp(s.pW, L.desc[L.pW].offset, L.desc[L.pW].size);
  cp(s.pB, L.desc[L.pB].offset, L.d.A1);
  cp(s.vW, L.desc[L.vW].offset, L.desc[L.vW].size);
  cp(s.vB, L.desc[L.vB].offset, L.d.FC);
  cp(s.voW, L.desc[L.voW].offset, L.desc[L.voW].size);
  cp(s.voB, L.desc[L.voB].offset, 1);
}

// ---------------------------------------------------------------------------------------------
// conv (cross-correlation, same padding) + BN-test affine + ReLU.  mode 0: out = y ;
// mode 1: out = relu(out + y) (second branch of a shared block, dual.go:67-73).
__global__ void k_unit_f32(const float* __restrict__ x, const float* __restrict__ filt, const float* __restrict__ gamma,
                           const float* __restrict__ beta, float* out, const int* __restrict__ n_dev, int n_max, int Ci,
                           int Co, int H, int W, int k, int mode) {
  const int n = min(*n_dev, n_max);
  const int HW = H * W;
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)n * Co * HW) return;
  const int hw = (int)(idx % HW), co = (int)((idx / HW) % Co), b = (int)(idx / ((size_t)HW * Co));
  const int y = hw / W, xx = hw - y * W, pad = (k - 1) / 2;
  const float* xb = x + (size_t)b * Ci * HW;
  const float* wk = filt + (size_t)co * Ci * k * k;
  float acc = 0.0f;
  for (int ci = 0; ci < Ci; ci++)
    for (int ky = 0; ky < k; ky++) {
      int yy = y + ky - pad;
      if (yy < 0 || yy >= H) continue;
      for (int kx = 0; kx < k; kx++) {
        int xc = xx + kx - pad;
        if (xc < 0 || xc >= W) continue;
        acc = __fadd_rn(acc, __fmul_rn(wk[(ci * k + ky) * k + kx], xb[(size_t)ci * HW + yy * W + xc]));
      }
    }
  const float s = __fsqrt_rn(__fadd_rn(0.0f, 1e-5f));  // sqrt(var + eps), var = 0 after BatchNormOp.Reset()
  float t = __fdiv_rn(acc, s);
  float v = __fadd_rn(__fmul_rn(gamma[co * HW + hw], t), beta[co * HW + hw]);
  v = v > 0.0f ? v : 0.0f;
  if (mode == 1) { float sum = __fadd_rn(out[idx], v); v = sum > 0.0f ? sum : 0.0f; }
  out[idx] = v;
}

// policy/value heads after the two 1x1 units: ph [n, 2*HW], vh [n, HW]
__global__ void k_heads_f32(const float* __restrict__ ph, const float* __restrict__ vh, const float* __restrict__ Wp,
                            const float* __restrict__ bp, const float* __restrict__ Wv, const float* __restrict__ bv,
                            const float* __restrict__ Wo, const float* __restrict__ bo, float* policy, int ldp, float* value,
                            const int* __restrict__ n_dev, int n_max, int HW, int A1, int FC) {
  extern __shared__ float sm[];  // logits[A1], h[FC]
  const int n = min(*n_dev, n_max);
  const int b = blockIdx.x;
  if (b >= n) return;
  float* logits = sm;
  float* h = sm + A1;
  const float* p = ph + (size_t)b * 2 * HW;
  const float* v = vh + (size_t)b * HW;
  for (int a = threadIdx.x; a < A1; a += blockDim.x) {
    float acc = 0.0f;
    for (int j = 0; j < 2 * HW; j++) acc = __fadd_rn(acc, __fmul_rn(p[j], Wp[(size_t)j * A1 + a]));
    logits[a] = expf(__fadd_rn(acc, bp[a]));  // SoftMax without max subtraction (dual.go:81)
  }
  for (int f = threadIdx.x; f < FC; f += blockDim.x) {
    float acc = 0.0f;
    for (int j = 0; j < HW; j++) acc = __fadd_rn(acc, __fmul_rn(v[j], Wv[(size_t)j * FC + f]));
    acc = __fadd_rn(acc, bv[f]);
    h[f] = acc > 0.0f ? acc : 0.0f;
  }
  __syncthreads();
  __shared__ float ssum;
  if (threadIdx.x == 0) {
    float s = 0.0f;
    for (int a = 0; a < A1; a++) s = __fadd_rn(s, logits[a]);
    ssum = s;
    float acc = 0.0f;
    for (int f = 0; f < FC; f++) acc = __fadd_rn(acc, __fmul_rn(h[f], Wo[f]));
    value[b] = tanhf(__fadd_rn(acc, bo[0]));
  }
  __syncthreads();
  for (int a = threadIdx.x; a < A1; a += blockDim.x) policy[(size_t)b * ldp + a] = __fdiv_rn(logits[a], ssum);
}

// Throughput version of the heads for the tensor-core path: SB samples per block share every weight
// load (the per-sample kernel above re-reads Policy_w from L2 for each sample).  Accumulation per
// output still runs in ascending j; the softmax sum and the final dot product use warp reductions.
template <int SB>
__global__ void k_heads_tiled(const float* __restrict__ ph, const float* __restrict__ vh, const float* __restrict__ Wp,
                              const float* __restrict__ bp, const float* __restrict__ Wv, const float* __restrict__ bv,
                              const float* __restrict__ Wo, const float* __restrict__ bo, float* policy, int ldp,
                              float* value, const int* __restrict__ n_dev, int n_max, int HW, int A1, int FC) {
  extern __shared__ float sm[];
  const int n = min(*n_dev, n_max);
  const int b0 = blockIdx.x * SB;
  if (b0 >= n) return;
  const int nb = min(SB, n - b0);
  const int J2 = 2 * HW;
  float* phs = sm;                  // [SB][2HW]
  float* vhs = phs + SB * J2;       // [SB][HW]
  float* lg = vhs + SB * HW;        // [SB][A1]
  float* hh = lg + SB * A1;         // [SB][FC]
  for (int i = threadIdx.x; i < SB * J2; i += blockDim.x) { int s = i / J2; phs[i] = s < nb ? ph[(size_t)b0 * J2 + i] : 0.0f; }
  for (int i = threadIdx.x; i < SB * HW; i += blockDim.x) { int s = i / HW; vhs[i] = s < nb ? vh[(size_t)b0 * HW + i] : 0.0f; }
  __syncthreads();
  for (int a = threadIdx.x; a < A1; a += blockDim.x) {
    float acc[SB];
#pragma unroll
    for (int s = 0; s < SB; s++) acc[s] = 0.0f;
    for (int j = 0; j < J2; j++) {
      const float w = __ldg(Wp + (size_t)j * A1 + a);
#pragma unroll
      for (int s = 0; s < SB; s++) acc[s] = fmaf(phs[s * J2 + j], w, acc[s]);
    }
    const float bias = bp[a];
#pragma unroll
    for (int s = 0; s < SB; s++) lg[s * A1 + a] = expf(acc[s] + bias);
  }
  for (int f = threadIdx.x; f < FC; f += blockDim.x) {
    float acc[SB];
#pragma unroll
    for (int s = 0; s < SB; s++) acc[s] = 0.0f;
    for (int j = 0; j < HW; j++) {
      const float w = __ldg(Wv + (size_t)j * FC + f);
#pragma unroll
      for (int s = 0; s < SB; s++) acc[s] = fmaf(vhs[s * HW + j], w, acc[s]);
    }
    const float bias = bv[f];
#pragma unroll
    for (int s = 0; s < SB; s++) { float v = acc[s] + bias; hh[s * FC + f] = v > 0.0f ? v : 0.0f; }
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int s = warp; s < nb; s += nw) {
    float sum = 0.0f, dot = 0.0f;
    for (int a = lane; a < A1; a += 32) sum += lg[s * A1 + a];
    for (int f = lane; f < FC; f += 32) dot = fmaf(hh[s * FC + f], Wo[f], dot);
#pragma unroll
    for (int off = 16; off; off >>= 1) { sum += __shfl_xor_sync(0xffffffffu, sum, off); dot += __shfl_xor_sync(0xffffffffu, dot, off); }
    for (int a = lane; a < A1; a += 32) policy[(size_t)(b0 + s) * ldp + a] = lg[s * A1 + a] / sum;
    if (lane == 0) value[b0 + s] = tanhf(dot + bo[0]);
  }
}

// per device, once per engine: opt-in maximum (engines of different head sizes share the function attribute)
void heads_tiled_configure() {
  int dev = 0, optin = 0;
  CUDA_CHECK(cudaGetDevice(&dev));
  CUDA_CHECK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  CUDA_CHECK(cudaFuncSetAttribute(k_heads_tiled<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, optin));
  CUDA_CHECK(cudaFuncSetAttribute(k_heads_tiled<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, optin));
  CUDA_CHECK(cudaFuncSetAttribute(k_heads_tiled<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, optin));
  CUDA_CHECK(cudaFuncSetAttribute(k_heads_tiled<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, optin));
}
template <int SB>
static void launch_heads_tiled(const NetDims& d, const Snapshot& s, const float* ph, const float* vh, const int* n_dev, int n_max,
                               float* policy, int ldp, float* value, cudaStream_t st) {
  const size_t sm = (size_t)SB * (3 * d.HW() + d.A1 + d.FC) * 4;
  k_heads_tiled<SB><<<(n_max + SB - 1) / SB, 256, sm, st>>>(ph, vh, s.d + s.pW, s.d + s.pB, s.d + s.vW, s.d + s.vB, s.d + s.voW,
                                                          s.d + s.voB, policy, ldp, value, n_dev, n_max, d.HW(), d.A1, d.FC); LAUNCH_CHECK();
}
// Samples per block: the most that still gives every SM a block (each sample's arithmetic does not depend on it)
void heads_tiled(const NetLayout& L, const Snapshot& s, const float* ph, const float* vh, const int* n_dev, int n_max,
                 float* policy, int ldp, float* value, cudaStream_t st, unsigned long long* launches) {
  const NetDims& d = L.d;
  static int num_sms = 0;
  if (!num_sms) { int dev = 0; CUDA_CHECK(cudaGetDevice(&dev)); CUDA_CHECK(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev)); }
  if (n_max >= 8 * num_sms) launch_heads_tiled<8>(d, s, ph, vh, n_dev, n_max, policy, ldp, value, st);
  else if (n_max >= 4 * num_sms) launch_heads_tiled<4>(d, s, ph, vh, n_dev, n_max, policy, ldp, value, st);
  else if (n_max >= 2 * num_sms) launch_heads_tiled<2>(d, s, ph, vh, n_dev, n_max, policy, ldp, value, st);
  else launch_heads_tiled<1>(d, s, ph, vh, n_dev, n_max, policy, ldp, value, st);
  if (launches) (*launches)++;
}

void fp32_scratch_alloc(Fp32Scratch& s, const NetDims& d, int n_max) {
  size_t act = (size_t)n_max * d.K * d.HW();
  CUDA_CHECK(cudaMalloc(&s.a, act * 4));
  CUDA_CHECK(cudaMalloc(&s.b, act * 4));
  CUDA_CHECK(cudaMalloc(&s.ph, (size_t)n_max * 2 * d.HW() * 4));
  CUDA_CHECK(cudaMalloc(&s.vh, (size_t)n_max * d.HW() * 4));
  s.cap = n_max;
}
void fp32_scratch_free(Fp32Scratch& s) {
  cudaFree(s.a); cudaFree(s.b); cudaFree(s.ph); cudaFree(s.vh);
  s = Fp32Scratch();
}

static void run_unit(const NetLayout& L, const Snapshot& s, int ui, const float* x, float* out, const int* n_dev, int n_max,
                     int mode, cudaStream_t st, unsigned long long* launches) {
  const SnapUnit& u = s.units[ui];
  size_t total = (size_t)n_max * u.Co * L.d.HW();
  int threads = 128;
  if ((total + threads - 1) / threads > 0x7fffffffull) throw std::runtime_error("k_unit_f32: batch x channels x points exceeds the grid limit");
  unsigned blocks = (unsigned)((total + threads - 1) / threads);
  k_unit_f32<<<blocks, threads, 0, st>>>(x, s.d + u.filter, s.d + u.gamma, s.d + u.beta, out, n_dev, n_max, u.Ci, u.Co,
                                         L.d.H, L.d.W, u.k, mode); LAUNCH_CHECK();
  if (launches) (*launches)++;
}

void heads_fp32(const NetLayout& L, const Snapshot& s, Fp32Scratch& sc, const float* tower, const int* n_dev, int n_max,
                float* policy, int ldp, float* value, cudaStream_t st, unsigned long long* launches) {
  const NetDims& d = L.d;
  int pu = 1 + 2 * d.SharedLayers, vu = pu + 1;
  run_unit(L, s, pu, tower, sc.ph, n_dev, n_max, 0, st, launches);
  run_unit(L, s, vu, tower, sc.vh, n_dev, n_max, 0, st, launches);
  size_t sm = (size_t)(d.A1 + d.FC) * 4;
  if (sm > 48 * 1024) throw std::runtime_error("k_heads_f32: ActionSpace + FC exceeds 48 KB of shared memory (use the tiled heads)");
  k_heads_f32<<<n_max, 128, sm, st>>>(sc.ph, sc.vh, s.d + s.pW, s.d + s.pB, s.d + s.vW, s.d + s.vB, s.d + s.voW,
                                      s.d + s.voB, policy, ldp, value, n_dev, n_max, d.HW(), d.A1, d.FC); LAUNCH_CHECK();
  if (launches) (*launches)++;
}

const float* forward_fp32(const NetLayout& L, const Snapshot& s, Fp32Scratch& sc, const float* planes, const int* n_dev, int n_max,
                          float* policy, int ldp, float* value, cudaStream_t st, unsigned long long* launches) {
  const NetDims& d = L.d;
  float* cur = sc.a;
  float* nxt = sc.b;
  run_unit(L, s, 0, planes, cur, n_dev, n_max, 0, st, launches);
  for (int i = 0; i < d.SharedLayers; i++) {
    run_unit(L, s, 1 + 2 * i, cur, nxt, n_dev, n_max, 0, st, launches);
    run_unit(L, s, 2 + 2 * i, cur, nxt, n_dev, n_max, 1, st, launches);
    float* t = cur; cur = nxt; nxt = t;
  }
  heads_fp32(L, s, sc, cur, n_dev, n_max, policy, ldp, value, st, launches);
  return cur;
}
