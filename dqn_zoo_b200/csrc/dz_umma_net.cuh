// The batch-32 learner step's torso and 512-wide FC layer on the TMA-fed tensor-core kernels (dz_umma.cuh):
// interface between dz_learner.cu and dz_umma_net.cu.  networks.py:181-204 (dqn_torso), :207-221 (dqn_value_head),
// :137-178 (noisy_linear), :224-261 (rainbow streams).
#pragma once
#include "dz_umma_host.cuh"

namespace dz {

struct UmNetDesc {
  int B, H, W;                       // batch, observation height / width (4 stacked frames)
  int npass;                         // network applies sharing one launch (2 or 3)
  int pass_target[3];                // 1: the pass uses the target parameters
  const float* online;
  const float* target;
  int64_t off_conv_w[3], off_conv_b[3];
  int use_fc;                        // the 3136 -> 512 layer(s) run here (everything but IQN)
  int nstream;                       // 1, or 2 for rainbow (adv, val)
  int noisy;                         // rainbow: mu + sigma weights, factorised noise
  int64_t off_fc_w[2], off_fc_b[2], off_fc_sw[2], off_fc_sb[2];
  int noise_apply[3];                // rainbow: noise apply index of each pass
  int64_t noise_stride;              // floats per apply
  int64_t noise_off_in[2], noise_off_out[2];   // offsets of eps_in[feat] / eps_out[512] of stream s inside one apply
  // 1: forward-only plan for acting (npass 1 on the online blob, any B up to the actor's cap): forward buffers and
  // launches only, the fc x operand in row chunks of 64 and split counts that depend on the geometry alone, so that
  // every row's arithmetic is the same at every B.
  int fwd_only;
};

struct UmNet;

// Geometry the path supports (else the learner keeps the fp32-FMA kernels).  The learner's plans take B <= 64;
// forward-only plans any B >= 1.
bool um_net_supported(const UmNetDesc& d);
int64_t um_net_workspace_bytes(const UmNetDesc& d);
// `base` may be nullptr (size query through carve); buffers are carved from it in a fixed order.
int um_net_create(const UmNetDesc& d, char* base, UmNet** out);
void um_net_destroy(UmNet* n);
void um_net_trace(UmNet* n, const char* tag, long long* d_trace);   // debug: clock stamps of CTA 0 of the launch `tag`
int um_net_mma_path(UmNet* n, const char* tag);   // UM_PATH_MMA_SYNC / UM_PATH_WGMMA of the launch `tag`; -1: no such launch

// Buffers the rest of the learner reads / writes (fp32 views of the activations and gradients).
float* um_act_f32(UmNet* n, int layer, int pass);      // layer 1..3 -> [B][h][w][C] (layers 1, 2: the tf32 hi image)
float* um_dact_f32(UmNet* n, int layer);               // layer 1..3: d loss / d (pre-ReLU masked) activation of pass 0
float* um_act_lo(UmNet* n, int layer);                 // layer 1, 2: tf32 lo image of pass 0's activation (hi: um_act_f32)
float* um_dact_hi(UmNet* n, int layer);                // layer 1..3: tf32 hi / lo of um_dact_f32, the operands of the next GEMM
float* um_dact_lo(UmNet* n, int layer);
float* um_h1_f32(UmNet* n, int pass, int stream);      // [B][512] (post-ReLU)
float* um_dh1_f32(UmNet* n, int stream);               // [B][512] gradient wrt h1 (already masked), INPUT of um_backward_fc
float* um_dh1_hi(UmNet* n, int stream);               // tf32 hi / lo of dh1 (written by the producer or by um_split_dh1)
float* um_dh1_lo(UmNet* n, int stream);

// One launch each unless noted.  rows[p]: row-pointer table of pass p (uint8 observations, gathered in place).
int um_pack_weights(UmNet* n, void* stream);                                   // conv weight images (both nets;
                                                                               // forward-only: online forward images)
int um_bind_noise(UmNet* n, const float* noise);                               // noisy fc: the noise buffer um_forward_fc
                                                                               // will read (synchronous; outside captures)
int um_forward_torso(UmNet* n, const uint8_t* const* const* rows, void* stream);   // conv1, conv2, conv3
int um_forward_fc(UmNet* n, const float* noise, void* stream);                 // fc1 / noisy1 + finish -> h1
int um_split_dh1(UmNet* n, void* stream);                                      // dh1 fp32 -> hi/lo (if the producer wrote fp32 only)
int um_backward_fc(UmNet* n, const float* noise, void* stream);                // fc1 / noisy1 input gradient + finish -> dact3
int um_split_dact3(UmNet* n, void* stream);                                    // dact3 fp32 -> hi/lo (IQN: produced by the Hadamard kernel)
int um_wgrad_conv1(UmNet* n, const uint8_t* const* rows0, void* stream);       // uint8 rows x dact1 -> one partial per CTA
int um_wgrad_conv3(UmNet* n, void* stream);                                    // act2 x dact3 -> split partials
int um_wgrad_conv2(UmNet* n, void* stream);                                    // act1 x dact2 -> split partials
int um_wgrad_finish_layer(UmNet* n, int layer, float* dW, float* db, float* norm_parts, void* stream);   // partial sums + bias gradient of
                                                                               // conv layer 1..3 (+ its split-norm partials)
int um_norm_slots(UmNet* n);                                                   // floats of the split-norm slot array
int um_backward_conv3(UmNet* n, void* stream);                                 // dact3 -> dact2
int um_backward_conv2(UmNet* n, void* stream);                                 // dact2 -> dact1

}  // namespace dz
