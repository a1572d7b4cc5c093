// agogo_b200 — K7: dual.Train (dualnet/meta.go:16-54) on the device, fp32 CUDA cores.
// One step = forward in BatchNorm train mode on a batch of exactly BatchSize samples, the
// reference's loss (dual.go:105-126: "xent" on raw logits, ermahagerdmonards.go:106-147, + MSE on
// the pre-tanh value), reverse-mode gradients for every Model() tensor (batch-shaped BN affines
// and biases included), vanilla SGD (meta.go:20,39).  fp32 throughout: shared-memory tiled implicit
// GEMMs for the three conv passes (4x4 register tiles), block reductions for BatchNorm, no atomics
// => deterministic; the tensor-core version of the conv passes is the next optimisation row.  Semantics are pinned against oracle/dual.hpp
// (dual_train_step), whose backward is itself pinned by a finite-difference check.
#include <algorithm>
#include <cstdlib>
#include <stdexcept>
#include <vector>

#include "nn.cuh"
#include "train.cuh"
#include "tower_tc.cuh"

namespace {

// ---- shared-memory tiled fp32 convolutions (used for every layer of the training pass) -------------
// Implicit GEMM  out[co, p] (+)= sum_q Wm[co, q] * im2col(x)[q, p],  q = (ci, ky, kx), p = (b, y, x):
// 64 output channels x 64 positions per block, 16x16 threads with a 4x4 register tile each, the
// reduction dimension streamed through shared memory in chunks of 8 input channels.
constexpr int TT = 64;   // tile edge (channels / positions)
constexpr int CKC = 8;   // input channels per chunk
template <bool ACC>
__global__ void __launch_bounds__(256) k_conv_fwd_tiled(const float* __restrict__ x, const float* __restrict__ w, float* out,
                                                        int B, int Ci, int Co, int H, int W, int k) {
  __shared__ float sW[CKC * 9][TT + 1];  // [q][co]
  __shared__ float sX[CKC * 9][TT];      // [q][p]
  const int HW = H * W, kk = k * k, pad = (k - 1) / 2;
  const int P = B * HW;
  const int p0 = blockIdx.x * TT, c0 = blockIdx.y * TT;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) acc[i][j] = 0.0f;
  for (int ci0 = 0; ci0 < Ci; ci0 += CKC) {
    const int nq = min(CKC, Ci - ci0) * kk;
    for (int e = threadIdx.x; e < nq * TT; e += 256) {
      const int q = e / TT, c = e - q * TT;
      const int ci = ci0 + q / kk, t = q - (q / kk) * kk;
      sW[q][c] = (c0 + c < Co) ? w[((size_t)(c0 + c) * Ci + ci) * kk + t] : 0.0f;
    }
    for (int e = threadIdx.x; e < nq * TT; e += 256) {
      const int q = e / TT, pp = e - q * TT;
      const int ci = ci0 + q / kk, t = q - (q / kk) * kk;
      const int p = p0 + pp;
      float v = 0.0f;
      if (p < P) {
        const int b = p / HW, hw = p - b * HW;
        const int yy = hw / W + t / k - pad, xx = hw % W + t % k - pad;
        if (yy >= 0 && yy < H && xx >= 0 && xx < W) v = x[((size_t)b * Ci + ci) * HW + yy * W + xx];
      }
      sX[q][pp] = v;
    }
    __syncthreads();
    for (int q = 0; q < nq; q++) {
      float wv[4], xv[4];
#pragma unroll
      for (int i = 0; i < 4; i++) wv[i] = sW[q][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; j++) xv[j] = sX[q][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = fmaf(wv[i], xv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int co = c0 + ty * 4 + i;
    if (co >= Co) continue;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int p = p0 + tx * 4 + j;
      if (p >= P) continue;
      const int b = p / HW, hw = p - b * HW;
      float* o = out + ((size_t)b * Co + co) * HW + hw;
      if (ACC) *o += acc[i][j]; else *o = acc[i][j];
    }
  }
}
// wt[ci][co][ky][kx] = w[co][ci][k-1-ky][k-1-kx]: backward-data is the forward kernel on the mirrored, transposed filter
__global__ void k_flip_filter(const float* __restrict__ w, float* wt, int Ci, int Co, int k) {
  const int kk = k * k;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= Ci * Co * kk) return;
  const int t = idx % kk, co = (idx / kk) % Co, ci = idx / (kk * Co);
  wt[idx] = w[((size_t)co * Ci + ci) * kk + (kk - 1 - t)];
}
// dW[co, (ci,t)] = sum_p dz[co, p] * x[ci, p + shift(t)]: 64 x 64 outputs per block, positions streamed in chunks of 32
__global__ void __launch_bounds__(256) k_conv_bwd_w_tiled(const float* __restrict__ x, const float* __restrict__ dz, float* dW,
                                                          int B, int Ci, int Co, int H, int W, int k) {
  constexpr int PK = 32;
  __shared__ float sD[PK][TT + 1];  // [p][co]
  __shared__ float sXs[PK][TT + 1]; // [p][(ci,t)]
  const int HW = H * W, kk = k * k, pad = (k - 1) / 2;
  const int P = B * HW, Q = Ci * kk;
  const int q0 = blockIdx.x * TT, c0 = blockIdx.y * TT;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  // blockIdx.z = slice of the position range (few-output layers would otherwise run on a handful of blocks);
  // slice z writes its partial to dW + z * Co * Q, k_sum_slices adds them in slice order
  const int chunk = ((P + gridDim.z - 1) / gridDim.z + PK - 1) / PK * PK;
  const int p_begin = blockIdx.z * chunk, p_end = min(P, p_begin + chunk);
  dW += (size_t)blockIdx.z * Co * Q;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) acc[i][j] = 0.0f;
  for (int pb = p_begin; pb < p_end; pb += PK) {
    for (int e = threadIdx.x; e < PK * TT; e += 256) {
      const int c = e / PK, pp = e - c * PK;  // consecutive threads walk positions: coalesced in hw
      const int p = pb + pp;
      float v = 0.0f;
      if (p < p_end && c0 + c < Co) { const int b = p / HW, hw = p - b * HW; v = dz[((size_t)b * Co + c0 + c) * HW + hw]; }
      sD[pp][c] = v;
    }
    for (int e = threadIdx.x; e < PK * TT; e += 256) {
      const int qq = e / PK, pp = e - qq * PK;
      const int q = q0 + qq, p = pb + pp;
      float v = 0.0f;
      if (p < p_end && q < Q) {
        const int ci = q / kk, t = q - ci * kk;
        const int b = p / HW, hw = p - b * HW;
        const int yy = hw / W + t / k - pad, xx = hw % W + t % k - pad;
        if (yy >= 0 && yy < H && xx >= 0 && xx < W) v = x[((size_t)b * Ci + ci) * HW + yy * W + xx];
      }
      sXs[pp][qq] = v;
    }
    __syncthreads();
#pragma unroll 4
    for (int pp = 0; pp < PK; pp++) {
      float dv[4], xv[4];
#pragma unroll
      for (int i = 0; i < 4; i++) dv[i] = sD[pp][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; j++) xv[j] = sXs[pp][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = fmaf(dv[i], xv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int co = c0 + ty * 4 + i;
    if (co >= Co) continue;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int q = q0 + tx * 4 + j;
      if (q < Q) dW[(size_t)co * Q + q] = acc[i][j];
    }
  }
}

__global__ void k_sum_slices(const float* __restrict__ part, int slices, size_t n, float* __restrict__ out) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  float acc = 0.0f;
  for (int z = 0; z < slices; z++) acc += part[(size_t)z * n + idx];
  out[idx] = acc;
}

__device__ inline float block_sum(float v, float* sh) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
#pragma unroll
  for (int off = 16; off; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  if (lane == 0) sh[warp] = v;
  __syncthreads();
  float r = 0.0f;
  if (threadIdx.x < 32) {
    r = threadIdx.x < nw ? sh[threadIdx.x] : 0.0f;
#pragma unroll
    for (int off = 16; off; off >>= 1) r += __shfl_xor_sync(0xffffffffu, r, off);
    if (threadIdx.x == 0) sh[0] = r;
  }
  __syncthreads();
  r = sh[0];
  __syncthreads();
  return r;
}

// per channel: mean and biased variance over (B, HW)
__global__ void k_bn_stats(const float* __restrict__ z, float* mean, float* var, int B, int Co, int HW) {
  __shared__ float sh[32];
  const int co = blockIdx.x;
  const int m = B * HW;
  float s = 0.0f;
  for (int i = threadIdx.x; i < m; i += blockDim.x) { int b = i / HW, hw = i - b * HW; s += z[((size_t)b * Co + co) * HW + hw]; }
  const float mu = block_sum(s, sh) / (float)m;
  float v = 0.0f;
  for (int i = threadIdx.x; i < m; i += blockDim.x) { int b = i / HW, hw = i - b * HW; float d = z[((size_t)b * Co + co) * HW + hw] - mu; v += d * d; }
  const float vv = block_sum(v, sh) / (float)m;
  if (threadIdx.x == 0) { mean[co] = mu; var[co] = vv; }
}
__global__ void k_bn_apply(const float* __restrict__ z, const float* __restrict__ mean, const float* __restrict__ var,
                           const float* __restrict__ gamma, const float* __restrict__ beta, float* xn, float* y, size_t total,
                           int Co, int HW) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int co = (int)((idx / HW) % Co);
  const float sd = sqrtf(var[co] + 1e-5f);
  const float n = (z[idx] - mean[co]) / sd;
  xn[idx] = n;
  const float v = gamma[idx] * n + beta[idx];
  y[idx] = v > 0.0f ? v : 0.0f;
}
__global__ void k_add_relu(const float* __restrict__ a, const float* __restrict__ b, float* out, size_t n) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  const float s = a[idx] + b[idx];
  out[idx] = s > 0.0f ? s : 0.0f;
}
// out[b,o] = sum_j in[b,j] W[j,o] + bias[b,o]  (batch-shaped bias, ermahagerdmonards.go:80-83)
__global__ void k_linear_fwd(const float* __restrict__ in, const float* __restrict__ Wm, const float* __restrict__ bias,
                             float* out, int B, int J, int O, int relu) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * O) return;
  const int b = idx / O, o = idx - b * O;
  float acc = 0.0f;
  for (int j = 0; j < J; j++) acc += in[(size_t)b * J + j] * Wm[(size_t)j * O + o];
  acc += bias[idx];
  out[idx] = relu ? (acc > 0.0f ? acc : 0.0f) : acc;
}
// cost + d cost/d logits + d cost/d vraw (dual.go:105-126)
__global__ void k_loss(const float* __restrict__ logits, const float* __restrict__ Pi, const float* __restrict__ vraw,
                       const float* __restrict__ V, float* dlog, float* dv, float* cost, int B, int A) {
  __shared__ float sh[32];
  const int n = B * A;
  float ps = 0.0f;
  const float invBA = 1.0f / (float)n;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    ps += -(Pi[i] * logits[i] + (1.0f - Pi[i]) * (1.0f - logits[i]));
    dlog[i] = (1.0f - 2.0f * Pi[i]) * invBA;
  }
  const float psum = block_sum(ps, sh);
  float vs = 0.0f;
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    float d = vraw[b] - V[b];
    vs += d * d;
    dv[b] = 2.0f * d / (float)B;
  }
  const float vsum = block_sum(vs, sh);
  if (threadIdx.x == 0) *cost = psum / (float)n + vsum / (float)B;
}
// dW[j,o] = sum_b in[b,j] dout[b,o]
__global__ void k_linear_bwd_w(const float* __restrict__ in, const float* __restrict__ dout, float* dW, int B, int J, int O) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= J * O) return;
  const int j = idx / O, o = idx - j * O;
  float acc = 0.0f;
  for (int b = 0; b < B; b++) acc += in[(size_t)b * J + j] * dout[(size_t)b * O + o];
  dW[idx] = acc;
}
// din[b,j] = sum_o W[j,o] dout[b,o]
__global__ void k_linear_bwd_in(const float* __restrict__ Wm, const float* __restrict__ dout, float* din, int B, int J, int O) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * J) return;
  const int b = idx / J, j = idx - b * J;
  float acc = 0.0f;
  for (int o = 0; o < O; o++) acc += Wm[(size_t)j * O + o] * dout[(size_t)b * O + o];
  din[idx] = acc;
}
__global__ void k_relu_mask(const float* __restrict__ act, float* d, size_t n) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx < n && !(act[idx] > 0.0f)) d[idx] = 0.0f;
}
// BN backward, part 1: ReLU gate, dgamma/dbeta (batch-shaped: one contribution each), dxn
__global__ void k_bn_bwd_pre(const float* __restrict__ dy, const float* __restrict__ y, const float* __restrict__ xn,
                             const float* __restrict__ gamma, float* dgamma, float* dbeta, float* dxn, size_t total) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const float d = y[idx] > 0.0f ? dy[idx] : 0.0f;
  dgamma[idx] = d * xn[idx];
  dbeta[idx] = d;
  dxn[idx] = d * gamma[idx];
}
// part 2: dz = (dxn - mean(dxn) - xn * mean(dxn*xn)) / sqrt(var + eps), per channel, in place
__global__ void k_bn_bwd_apply(float* dxn, const float* __restrict__ xn, const float* __restrict__ var, int B, int Co, int HW) {
  __shared__ float sh[32];
  const int co = blockIdx.x;
  const int m = B * HW;
  float s1 = 0.0f, s2 = 0.0f;
  for (int i = threadIdx.x; i < m; i += blockDim.x) {
    int b = i / HW, hw = i - b * HW;
    size_t idx = ((size_t)b * Co + co) * HW + hw;
    s1 += dxn[idx];
    s2 += dxn[idx] * xn[idx];
  }
  const float m1 = block_sum(s1, sh) / (float)m;
  const float m2 = block_sum(s2, sh) / (float)m;
  const float sd = sqrtf(var[co] + 1e-5f);
  for (int i = threadIdx.x; i < m; i += blockDim.x) {
    int b = i / HW, hw = i - b * HW;
    size_t idx = ((size_t)b * Co + co) * HW + hw;
    dxn[idx] = (dxn[idx] - m1 - xn[idx] * m2) / sd;
  }
}
__global__ void k_sgd(float* p, const float* __restrict__ g, float lr, float gscale, size_t n) {
  const size_t n4 = n >> 2;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
    float4 pv = reinterpret_cast<float4*>(p)[i];
    const float4 gv = reinterpret_cast<const float4*>(g)[i];
    pv.x = pv.x - lr * (gv.x * gscale); pv.y = pv.y - lr * (gv.y * gscale);
    pv.z = pv.z - lr * (gv.z * gscale); pv.w = pv.w - lr * (gv.w * gscale);
    reinterpret_cast<float4*>(p)[i] = pv;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) { const size_t i = (n4 << 2) + threadIdx.x; p[i] = p[i] - lr * (g[i] * gscale); }
}

inline unsigned nblk(size_t n, int t = 256) { return (unsigned)((n + t - 1) / t); }

}  // namespace

// how many position slices the fp32 backward-filter kernel of a unit is launched with (1 = write dW directly)
// (sized for H100's 132 SMs: a layer with fewer blocks than SMs is sliced to about two blocks per SM)
static int dw_slices(const UnitH& u, int P) {
  const int blocks = ((u.Ci * u.k * u.k + TT - 1) / TT) * ((u.Co + TT - 1) / TT);
  if (blocks >= 132) return 1;
  return std::max(1, std::min({(264 + blocks - 1) / blocks, 64, (P + 255) / 256}));
}

struct TrainImpl {
  NetDims d;
  std::vector<float*> z, xn, y;   // per unit
  std::vector<float*> mean, var;  // per unit
  std::vector<float*> cur;        // block inputs/outputs: cur[0] = init output, cur[i+1] = block i output
  float *X = nullptr, *Pi = nullptr, *V = nullptr;
  float *logits = nullptr, *h1 = nullptr, *vraw = nullptr, *dlog = nullptr, *dv = nullptr, *dh1 = nullptr;
  float *dph = nullptr, *dvh = nullptr, *dcur = nullptr, *dprev = nullptr, *tmp = nullptr, *dl = nullptr;
  float* cost = nullptr;
  float* grads = nullptr;
  float* wflip = nullptr;  // mirrored/transposed filter of the unit being back-propagated
  float* dwpart = nullptr; // position-sliced partial filter gradients of the few-output layers
  size_t dwpart_n = 0;
  TcGemm tc;               // 3x3 forward / backward-data convs on wgmma (K in {64,128,256}); impl == nullptr -> fp32 tiled
  std::vector<void*> allocs;
  float* alloc(size_t n) {
    float* p;
    CUDA_CHECK(cudaMalloc(&p, std::max<size_t>(n, 1) * 4));
    allocs.push_back(p);
    return p;
  }
};

void train_ws_alloc(TrainWS& ws, const NetLayout& L) {
  if (ws.impl) return;
  TrainImpl* T = new TrainImpl;
  ws.impl = T;
  const NetDims& d = L.d;
  T->d = d;
  const size_t B = d.B, HW = d.HW();
  for (const UnitH& u : L.units) {
    size_t n = B * u.Co * HW;
    T->z.push_back(T->alloc(n)); T->xn.push_back(T->alloc(n)); T->y.push_back(T->alloc(n));
    T->mean.push_back(T->alloc(u.Co)); T->var.push_back(T->alloc(u.Co));
  }
  const size_t act = B * d.K * HW;
  for (int i = 0; i <= d.SharedLayers; i++) T->cur.push_back(i == 0 ? nullptr : T->alloc(act));
  T->X = T->alloc(B * d.F * HW); T->Pi = T->alloc(B * d.A1); T->V = T->alloc(B);
  T->logits = T->alloc(B * d.A1); T->h1 = T->alloc(B * d.FC); T->vraw = T->alloc(B);
  T->dlog = T->alloc(B * d.A1); T->dv = T->alloc(B); T->dh1 = T->alloc(B * d.FC);
  T->dph = T->alloc(B * 2 * HW); T->dvh = T->alloc(B * HW);
  T->dcur = T->alloc(act); T->dprev = T->alloc(act); T->tmp = T->alloc(act); T->dl = T->alloc(act);
  T->cost = T->alloc(1);
  { size_t mx = 1; for (const UnitH& u : L.units) mx = std::max(mx, (size_t)u.Ci * u.Co * u.k * u.k); T->wflip = T->alloc(mx); }
  for (const UnitH& u : L.units) {
    int slices = dw_slices(u, (int)(B * HW));
    if (slices > 1) T->dwpart_n = std::max(T->dwpart_n, (size_t)slices * u.Co * u.Ci * u.k * u.k);
  }
  if (T->dwpart_n) T->dwpart = T->alloc(T->dwpart_n);
  {
    const char* e = getenv("AZ_TRAIN_TC");
    if (tc_gemm_supported(d) && !(e && e[0] == '0')) tc_gemm_create(T->tc, d, d.B);
  }
  T->grads = T->alloc(L.total + 4);  // +4: the fused collective moves float4s
  CUDA_CHECK(cudaMemset(T->grads, 0, (L.total + 4) * 4));
}
void train_ws_free(TrainWS& ws) {
  TrainImpl* T = (TrainImpl*)ws.impl;
  if (!T) return;
  for (void* p : T->allocs) cudaFree(p);
  tc_gemm_destroy(T->tc);
  delete T;
  ws.impl = nullptr;
}
float* train_ws_grads(TrainWS& ws) { return ((TrainImpl*)ws.impl)->grads; }
float* train_ws_cost(TrainWS& ws) { return ((TrainImpl*)ws.impl)->cost; }
void train_ws_inputs(TrainWS& ws, float** X, float** Pi, float** V) {
  TrainImpl* T = (TrainImpl*)ws.impl;
  *X = T->X; *Pi = T->Pi; *V = T->V;
}

// forward + backward: fills grads (every Model() tensor gets exactly one contribution) and cost
void train_step_grads(TrainWS& ws, const NetLayout& L, const float* P, cudaStream_t st, unsigned long long* launches) {
  TrainImpl* T = (TrainImpl*)ws.impl;
  const NetDims& d = L.d;
  const int B = d.B, H = d.H, W = d.W, HW = d.HW(), K = d.K, A = d.A1, FC = d.FC;
  const int Lr = d.SharedLayers, pu = 1 + 2 * Lr, vu = pu + 1;
  auto Pp = [&](int i) { return P + L.desc[i].offset; };
  auto Gp = [&](int i) { return T->grads + L.desc[i].offset; };
  unsigned long long nl = 0;
  // same_x: x is the tensor the previous tensor-core call of this pass staged (the second branch of a block)
  auto unit_fwd = [&](int ui, const float* x, bool same_x = false) {
    const UnitH& u = L.units[ui];
    size_t n = (size_t)B * u.Co * HW;
    if (T->tc.impl && u.k == 3 && u.Co % 64 == 0)
      tc_gemm_conv(T->tc, x, u.Ci, Pp(u.filter), u.Co, u.Ci, false, T->z[ui], u.Co, false, 0,
                   same_x ? TC_OPERAND_REUSE : TC_OPERAND_PACK, st, &nl);
    else
      k_conv_fwd_tiled<false><<<dim3((B * HW + TT - 1) / TT, (u.Co + TT - 1) / TT), 256, 0, st>>>(x, Pp(u.filter), T->z[ui], B, u.Ci, u.Co, H, W, u.k); LAUNCH_CHECK();
    k_bn_stats<<<u.Co, 1024, 0, st>>>(T->z[ui], T->mean[ui], T->var[ui], B, u.Co, HW); LAUNCH_CHECK();
    k_bn_apply<<<nblk(n), 256, 0, st>>>(T->z[ui], T->mean[ui], T->var[ui], Pp(u.gamma), Pp(u.beta), T->xn[ui], T->y[ui], n, u.Co, HW); LAUNCH_CHECK();
    nl += 3;
  };
  // ---- forward
  unit_fwd(0, T->X);
  const float* cur = T->y[0];
  const size_t act = (size_t)B * K * HW;
  for (int i = 0; i < Lr; i++) {
    unit_fwd(1 + 2 * i, cur);
    unit_fwd(2 + 2 * i, cur, true);
    k_add_relu<<<nblk(act), 256, 0, st>>>(T->y[1 + 2 * i], T->y[2 + 2 * i], T->cur[i + 1], act); LAUNCH_CHECK();
    nl++;
    cur = T->cur[i + 1];
  }
  unit_fwd(pu, cur);
  unit_fwd(vu, cur);
  k_linear_fwd<<<nblk((size_t)B * A), 256, 0, st>>>(T->y[pu], Pp(L.pW), Pp(L.pB), T->logits, B, 2 * HW, A, 0); LAUNCH_CHECK();
  k_linear_fwd<<<nblk((size_t)B * FC), 256, 0, st>>>(T->y[vu], Pp(L.vW), Pp(L.vB), T->h1, B, HW, FC, 1); LAUNCH_CHECK();
  k_linear_fwd<<<nblk(B), 256, 0, st>>>(T->h1, Pp(L.voW), Pp(L.voB), T->vraw, B, FC, 1, 0); LAUNCH_CHECK();
  k_loss<<<1, 256, 0, st>>>(T->logits, T->Pi, T->vraw, T->V, T->dlog, T->dv, T->cost, B, A); LAUNCH_CHECK();
  nl += 4;
  // ---- backward: heads
  CUDA_CHECK(cudaMemcpyAsync(Gp(L.pB), T->dlog, (size_t)B * A * 4, cudaMemcpyDeviceToDevice, st));
  k_linear_bwd_w<<<nblk((size_t)2 * HW * A), 256, 0, st>>>(T->y[pu], T->dlog, Gp(L.pW), B, 2 * HW, A); LAUNCH_CHECK();
  k_linear_bwd_in<<<nblk((size_t)B * 2 * HW), 256, 0, st>>>(Pp(L.pW), T->dlog, T->dph, B, 2 * HW, A); LAUNCH_CHECK();
  CUDA_CHECK(cudaMemcpyAsync(Gp(L.voB), T->dv, (size_t)B * 4, cudaMemcpyDeviceToDevice, st));
  k_linear_bwd_w<<<nblk(FC), 256, 0, st>>>(T->h1, T->dv, Gp(L.voW), B, FC, 1); LAUNCH_CHECK();
  k_linear_bwd_in<<<nblk((size_t)B * FC), 256, 0, st>>>(Pp(L.voW), T->dv, T->dh1, B, FC, 1); LAUNCH_CHECK();
  k_relu_mask<<<nblk((size_t)B * FC), 256, 0, st>>>(T->h1, T->dh1, (size_t)B * FC); LAUNCH_CHECK();
  CUDA_CHECK(cudaMemcpyAsync(Gp(L.vB), T->dh1, (size_t)B * FC * 4, cudaMemcpyDeviceToDevice, st));
  k_linear_bwd_w<<<nblk((size_t)HW * FC), 256, 0, st>>>(T->y[vu], T->dh1, Gp(L.vW), B, HW, FC); LAUNCH_CHECK();
  k_linear_bwd_in<<<nblk((size_t)B * HW), 256, 0, st>>>(Pp(L.vW), T->dh1, T->dvh, B, HW, FC); LAUNCH_CHECK();
  nl += 7;
  // ---- backward: units
  auto unit_bwd = [&](int ui, const float* x, const float* dy, float* dx, bool same_x = false) {
    const UnitH& u = L.units[ui];
    size_t n = (size_t)B * u.Co * HW;
    k_bn_bwd_pre<<<nblk(n), 256, 0, st>>>(dy, T->y[ui], T->xn[ui], Pp(u.gamma), Gp(u.gamma), Gp(u.beta), T->tmp, n); LAUNCH_CHECK();
    k_bn_bwd_apply<<<u.Co, 1024, 0, st>>>(T->tmp, T->xn[ui], T->var[ui], B, u.Co, HW); LAUNCH_CHECK();
    const bool dw_tc = T->tc.impl && u.k == 3 && u.Ci == K && u.Co == K;
    if (dw_tc)
      tc_gemm_dw(T->tc, x, T->tmp, Gp(u.filter), same_x ? TC_OPERAND_REUSE : TC_OPERAND_PACK, st, &nl);
    else {
      const int slices = dw_slices(u, B * HW);
      const size_t nw = (size_t)u.Co * u.Ci * u.k * u.k;
      k_conv_bwd_w_tiled<<<dim3((u.Ci * u.k * u.k + TT - 1) / TT, (u.Co + TT - 1) / TT, slices), 256, 0, st>>>(
          x, T->tmp, slices > 1 ? T->dwpart : Gp(u.filter), B, u.Ci, u.Co, H, W, u.k); LAUNCH_CHECK();
      if (slices > 1) { k_sum_slices<<<nblk(nw), 256, 0, st>>>(T->dwpart, slices, nw, Gp(u.filter)); LAUNCH_CHECK(); nl++; }
    }
    nl += 3;
    if (dx && T->tc.impl && u.k == 3 && u.Ci % 64 == 0 && u.Co % 64 == 0) {
      // dz = T->tmp: its exponent was computed by the backward-filter call just above
      tc_gemm_conv(T->tc, T->tmp, u.Co, Pp(u.filter), u.Co, u.Ci, true, dx, u.Ci, true, 1,
                   dw_tc ? TC_OPERAND_PACK_KEEP_EXP : TC_OPERAND_PACK, st, &nl);
    } else if (dx) {  // dx += conv(dz, mirrored transposed filter)
      k_flip_filter<<<nblk((size_t)u.Ci * u.Co * u.k * u.k), 256, 0, st>>>(Pp(u.filter), T->wflip, u.Ci, u.Co, u.k); LAUNCH_CHECK();
      k_conv_fwd_tiled<true><<<dim3((B * HW + TT - 1) / TT, (u.Ci + TT - 1) / TT), 256, 0, st>>>(T->tmp, T->wflip, dx, B, u.Co, u.Ci, H, W, u.k); LAUNCH_CHECK();
      nl += 2;
    }
  };
  CUDA_CHECK(cudaMemsetAsync(T->dcur, 0, act * 4, st));
  unit_bwd(pu, cur, T->dph, T->dcur);
  unit_bwd(vu, cur, T->dvh, T->dcur);
  for (int i = Lr - 1; i >= 0; i--) {
    // out = relu(l1 + l2): gate on the block output
    CUDA_CHECK(cudaMemcpyAsync(T->dl, T->dcur, act * 4, cudaMemcpyDeviceToDevice, st));
    k_relu_mask<<<nblk(act), 256, 0, st>>>(T->cur[i + 1], T->dl, act); LAUNCH_CHECK();
    nl++;
    CUDA_CHECK(cudaMemsetAsync(T->dprev, 0, act * 4, st));
    const float* xin = i == 0 ? T->y[0] : T->cur[i];
    unit_bwd(1 + 2 * i, xin, T->dl, T->dprev);
    unit_bwd(2 + 2 * i, xin, T->dl, T->dprev, true);
    std::swap(T->dcur, T->dprev);
  }
  unit_bwd(0, T->X, T->dcur, nullptr);
  if (launches) *launches += nl;
}

// K8: gradient all-reduce fused with the SGD step, over NVLink peer memory (no NCCL on this path).
// Every rank runs this kernel on its own stream after its backward pass.  One-shot algorithm sized
// for NVSwitch (every peer at full bandwidth): rank r owns the r-th slice of the flat Model()
// buffer; it sums that slice of every rank's gradient straight out of peer HBM (fixed rank order,
// so the result is deterministic and — being computed once — identical everywhere), applies
// w -= lr * g / world to its slice and writes the updated slice into every rank's parameter buffer.
// Cross-GPU ordering uses epoch flags in peer memory: (A) "my gradients are complete" before anyone
// reads them, (B) "my slice is written everywhere" before anyone's next kernel may start.
__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// bounded spin on a peer-written epoch flag: false when the peer has not shown up within timeout_ns
__device__ __forceinline__ bool wait_epoch(volatile int* flag, int epoch, unsigned long long timeout_ns) {
  const unsigned long long t0 = global_ns();
  while (*flag < epoch) {
    if (global_ns() - t0 > timeout_ns) return false;
  }
  return true;
}
template <int WORLD>  // compile-time world size (0 = runtime): lets every peer load of a thread be issued up front
__global__ void k_allreduce_sgd_p2p(float* const* __restrict__ peer_grads, float* const* __restrict__ peer_params,
                                    int* const* __restrict__ peer_flags, int* my_flags, int rank, int world_rt, size_t n,
                                    float lr_over_world, int epoch, unsigned int* done_counter, unsigned long long timeout_ns,
                                    int* err) {
  const int world = WORLD ? WORLD : world_rt;
  __shared__ int s_last, s_ok;
  if (threadIdx.x == 0) s_ok = 1;
  __syncthreads();
  // (A) publish "gradients ready", then wait for everybody's
  if (blockIdx.x == 0 && threadIdx.x < world) {
    __threadfence_system();
    ((volatile int*)peer_flags[threadIdx.x])[rank] = epoch;
  }
  if (threadIdx.x < world) {
    if (!wait_epoch((volatile int*)my_flags + threadIdx.x, epoch, timeout_ns)) s_ok = 0;
  }
  __syncthreads();
  if (!s_ok) {  // a peer never arrived: report instead of spinning on the GPU forever; parameters are left untouched
    if (threadIdx.x == 0) atomicOr(err, ERR_COMM_TIMEOUT);
    return;
  }
  __threadfence_system();
  const size_t shard = (((n + world - 1) / world) + 3) & ~(size_t)3;
  const size_t lo = (size_t)rank * shard;
  const size_t hi = lo + shard < n ? lo + shard : ((n + 3) & ~(size_t)3);  // buffers are padded to a multiple of 4
  float* mine = peer_params[rank];
  float* pg[WORLD ? WORLD : 16];
  float* pp[WORLD ? WORLD : 16];
#pragma unroll
  for (int r = 0; r < (WORLD ? WORLD : 16); r++) { pg[r] = r < world ? peer_grads[r] : nullptr; pp[r] = r < world ? peer_params[r] : nullptr; }
  // peer loads cost ~2 us each: keep U x world 16-byte loads in flight per thread before touching the data
  constexpr int U = 4;
  const size_t stride = (size_t)gridDim.x * blockDim.x * 4;
  for (size_t i0 = lo + ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 4; i0 < hi; i0 += stride * U) {
    float4 g[U], p[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t i = i0 + (size_t)u * stride;
      g[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (i < hi) {
        p[u] = *reinterpret_cast<const float4*>(mine + i);
#pragma unroll
        for (int r = 0; r < (WORLD ? WORLD : 16); r++) {
          if (r < world) {
            const float4 v = *reinterpret_cast<const float4*>(pg[r] + i);
            g[u].x += v.x; g[u].y += v.y; g[u].z += v.z; g[u].w += v.w;
          }
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t i = i0 + (size_t)u * stride;
      if (i < hi) {
        float4 q = p[u];
        q.x -= lr_over_world * g[u].x; q.y -= lr_over_world * g[u].y; q.z -= lr_over_world * g[u].z; q.w -= lr_over_world * g[u].w;
#pragma unroll
        for (int r = 0; r < (WORLD ? WORLD : 16); r++)
          if (r < world) *reinterpret_cast<float4*>(pp[r] + i) = q;
      }
    }
  }
  // (B) the last block of this rank publishes "slice written" and waits for everybody's
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(done_counter, 1u) == gridDim.x - 1);
  __syncthreads();
  if (s_last) {
    if (threadIdx.x < world) {
      ((volatile int*)peer_flags[threadIdx.x])[world + rank] = epoch;
      if (!wait_epoch((volatile int*)my_flags + world + threadIdx.x, epoch, timeout_ns)) atomicOr(err, ERR_COMM_TIMEOUT);
    }
    if (threadIdx.x == 0) *done_counter = 0;
  }
}

void train_allreduce_sgd_p2p(float* const* peer_grads, float* const* peer_params, int* const* peer_flags, int* my_flags,
                             int rank, int world, size_t n, float lr, int epoch, unsigned int* done_counter, int num_sms,
                             int* err, cudaStream_t st, unsigned long long* launches) {
  static unsigned long long timeout_ns = 0;
  if (!timeout_ns) {
    const char* t = getenv("AZ_COMM_TIMEOUT_S");
    const double sec = t ? atof(t) : 60.0;
    timeout_ns = (unsigned long long)((sec > 0 ? sec : 60.0) * 1e9);
  }
  const size_t shard = (((n + world - 1) / world) + 3) & ~(size_t)3;
  int blocks = (int)std::min<size_t>((shard / 4 + 255) / 256, (size_t)num_sms * 8);
  if (blocks < 1) blocks = 1;
  if (world > 16) throw std::runtime_error("k_allreduce_sgd_p2p: world > 16");
#define AZ_LAUNCH_K8(W) k_allreduce_sgd_p2p<W><<<blocks, 256, 0, st>>>(peer_grads, peer_params, peer_flags, my_flags, rank, world, n, \
                                                                       lr / (float)world, epoch, done_counter, timeout_ns, err)
  if (world == 2) AZ_LAUNCH_K8(2);
  else if (world == 4) AZ_LAUNCH_K8(4);
  else if (world == 8) AZ_LAUNCH_K8(8);
  else AZ_LAUNCH_K8(0);
#undef AZ_LAUNCH_K8
  LAUNCH_CHECK();
  if (launches) (*launches)++;
}

void train_sgd(TrainWS& ws, const NetLayout& L, float* P, float lr, float gscale, cudaStream_t st, unsigned long long* launches) {
  TrainImpl* T = (TrainImpl*)ws.impl;
  k_sgd<<<(unsigned)std::min<size_t>((L.total / 4 + 255) / 256 + 1, 132 * 16), 256, 0, st>>>(P, T->grads, lr, gscale, L.total); LAUNCH_CHECK();
  if (launches) (*launches)++;
}
