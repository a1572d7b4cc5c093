// agogo_b200 — dual network: parameter layout and forward interfaces shared by engine.cu,
// nn_fp32.cu and tower_tc.cu.
//
// Canonical definition of dualnet.Dual (dualnet/dual.go:50-103, ermahagerdmonards.go) used by
// engine and oracle alike — see DESIGN.md "dualnet semantics" for the named assumptions about
// gorgonia's BatchNorm (full-shape learnable scale/bias; test mode after Reset => x/sqrt(eps)):
//   unit(x)  = relu( gamma ⊙ (conv(x, filter) / sqrt(eps)) + beta )        gamma,beta: [C,H,W] (batch row 0)
//   tower    = unit_init ; then SharedLayers x  relu(unit_a(x) + unit_b(x))  (no identity skip)
//   policy   = softmax( flatten(unit_1x1(K->2)) @ Policy_w + Policy_b[0] )
//   value    = tanh( relu(flatten(unit_1x1(K->1)) @ Value_w + Value_b[0]) @ ValueOutput_w + ValueOutput_b[0] )
#pragma once
#include <string>
#include <vector>

#include "common.cuh"

struct NetDims {
  int K, SharedLayers, FC, B /*train batch*/, W, H, F, A1 /*action_space*/;
  int HW() const { return W * H; }
};

struct ParamDescH {
  std::string name;
  int rank;
  int shape[4];
  size_t offset, size;
  int init;  // 0 zeros, 1 GlorotU(1.0), 2 GlorotN(1.0)
};
struct UnitH { int filter, gamma, beta, Ci, Co, k; };
struct NetLayout {
  NetDims d;
  std::vector<ParamDescH> desc;  // dual.Model() order
  std::vector<UnitH> units;      // Init, (Layer1, Layer2) x SharedLayers, PolicyHead, ValueHead
  int pW, pB, vW, vB, voW, voB;
  size_t total = 0;
};
NetLayout build_layout(const NetDims& d);
void init_params_host(const NetLayout& L, uint64_t seed, std::vector<float>* out);

// Inference snapshot of one agent (dual.Infer, meta.go:125-146): filters + batch row 0 of every
// batch-shaped tensor, flat on the device.  Offsets in floats.
struct SnapUnit { size_t filter, gamma, beta; int Ci, Co, k; };
struct Snapshot {
  float* d = nullptr;  // device
  size_t total = 0;
  std::vector<SnapUnit> units;
  size_t pW, pB, vW, vB, voW, voB;
};
Snapshot make_snapshot_layout(const NetLayout& L);
// gather train-form params (device) into the snapshot (device)
void snapshot_gather(const NetLayout& L, const float* params_dev, Snapshot& s, cudaStream_t st);

// fp32 CUDA-core forward (validation-grade, op order identical to the oracle's):
//   planes [n, F, H, W] (device) -> policy [n, ldp] (first A1 entries), value [n]
// n is read from *n_dev (device) and clamped to n_max.  Returns the tower output it handed to the heads (dense NCHW, in sc).
struct Fp32Scratch { float *a = nullptr, *b = nullptr, *ph = nullptr, *vh = nullptr; size_t cap = 0; };
void fp32_scratch_alloc(Fp32Scratch& s, const NetDims& d, int n_max);
void fp32_scratch_free(Fp32Scratch& s);
const float* forward_fp32(const NetLayout& L, const Snapshot& s, Fp32Scratch& sc, const float* planes, const int* n_dev, int n_max,
                          float* policy, int ldp, float* value, cudaStream_t st, unsigned long long* launches);
// heads only, from a dense fp32 NCHW tower output
void heads_fp32(const NetLayout& L, const Snapshot& s, Fp32Scratch& sc, const float* tower, const int* n_dev, int n_max,
                float* policy, int ldp, float* value, cudaStream_t st, unsigned long long* launches);
// heads from the post-1x1-unit activations ph [n,2*HW], vh [n,HW]: throughput version (SB samples per block)
void heads_tiled_configure();
void heads_tiled(const NetLayout& L, const Snapshot& s, const float* ph, const float* vh, const int* n_dev, int n_max,
                 float* policy, int ldp, float* value, cudaStream_t st, unsigned long long* launches);
