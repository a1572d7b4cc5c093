// agogo_b200 — wgmma/TMA residual tower (K5) interface.
#pragma once
#include "nn.cuh"

struct TcTower {
  bool ready = false;
  void* impl = nullptr;
};
// shapes the tensor-core tower handles (K multiple of 64, board fits the padded tiling); smaller
// nets (tic-tac-toe K=3, Connect-4 K=16) run on the fp32 CUDA-core kernels.
bool tc_tower_supported(const NetDims& d);
// fp16: AZ_FLAG_FP16_TOWER — activations and filters stored as one fp16 each, one wgmma pass (no lo buffers are allocated)
void tc_tower_alloc(TcTower& t, const NetDims& d, int n_max, int act_scale_log2, bool fp16);
// which kernel runs the fused layers (bench labels): 0 = k_conv3x3_tc (wgmma, 3 x fp16), 5 = k_net_small (the whole tower
// of a K = 64 net in one kernel), 6 = k_conv3x3_tc single fp16 plane, 7 = k_smallnet_fp16; -1 = no tensor-core tower
int tc_tower_kernel_kind(const TcTower& t);
void tc_tower_free(TcTower& t);
// split/scale/reorder the snapshot's filters and BN affines into the tensor-core operand layout
void tc_tower_prepare(TcTower& t, const Snapshot& s, cudaStream_t st);
// event timing of the fused-block conv launches (bench roofline); collect() synchronises the stream
void tc_tower_profile(TcTower& t, bool enable);
void tc_tower_profile_collect(TcTower& t, cudaStream_t st, double* conv_ms, double* conv_launches, double* fwd_ms,
                              double* fwd_calls);
void tc_tower_forward(TcTower& t, const NetLayout& L, const Snapshot& s, Fp32Scratch& sc, const float* planes,
                      const int* n_dev, int n_max, float* policy, int ldp, float* value, int* err_flag, cudaStream_t st,
                      unsigned long long* launches);
// diagnostics: the tower output of the last tc_tower_forward (the buffer the head convs read) as fp32 NCHW out [n][K][H][W]
void tc_tower_output(TcTower& t, const int* n_dev, int n_max, float* out, cudaStream_t st);

// K7: the 3x3 convolutions of the training pass (forward, backward-data, backward-filter) on wgmma (train_tc.cu)
struct TcGemm { void* impl = nullptr; };
enum {
  TC_OPERAND_PACK = 0,           // absmax -> exponent, split into fp16 hi/lo into the slot
  TC_OPERAND_PACK_KEEP_EXP = 1,  // split with the exponent the slot already holds (same tensor seen by an earlier call)
  TC_OPERAND_REUSE = 2,          // the slot already holds this tensor
};
bool tc_gemm_supported(const NetDims& d);
void tc_gemm_create(TcGemm& g, const NetDims& d, int B);
void tc_gemm_destroy(TcGemm& g);
// out[B][Cout][HW] (+)= conv3x3(x[B][Cin][HW], filter[fCo][fCi][3][3]); flip = backward-data (x = dz, Cin = fCo, Cout = fCi).
// x is staged in operand slot a_slot (0: activations, 1: gradients) according to a_state.
void tc_gemm_conv(TcGemm& g, const float* x, int Cin, const float* filter, int fCo, int fCi, bool flip, float* out, int Cout,
                  bool accumulate, int a_slot, int a_state, cudaStream_t st, unsigned long long* launches);
// dW[K][K][3][3] = sum over batch and positions of dz (x) shifted x  (backward-filter of a K->K 3x3 layer); x via slot 0,
// the exponent of dz is left in slot 1
void tc_gemm_dw(TcGemm& g, const float* x, const float* dz, float* dW, int x_state, cudaStream_t st, unsigned long long* launches);
