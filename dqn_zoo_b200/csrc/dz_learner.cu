// Learner half of the hot path: the jitted `update` of every dqn_zoo agent as hand-written CUDA.
//
//   networks      networks.py:58-363   (Nature-CNN torso, DQN / C51 / QR / IQN / Rainbow heads)
//   loss_fn       dqn/agent.py:85-107, double_q/agent.py:85-111, prioritized/agent.py:86-113,
//                 c51/agent.py:87-107, qrdqn/agent.py:88-110, rainbow/agent.py:85-109, iqn/agent.py:178-214
//   rlax 0.1.2    q_learning, double_q_learning, clip_gradient, l2_loss, categorical_l2_project,
//                 categorical_[double_]q_learning, quantile_q_learning (restated; SURVEY §8(c))
//   optax 0.1.2   adam, rmsprop(centered), clip_by_global_norm, apply_updates
//   _learn glue   rainbow/agent.py:181-198, prioritized/agent.py:187-206
//   munchausen    Munchausen DQN and Munchausen-IQN (Vieillard, Pietquin & Geist, NeurIPS 2020), outside the
//                 reference: dqn's / iqn's network with online(s_tm1) | target(s_tm1) | target(s_t) (DESIGN.md §13, §14)
//   fqf           Fully parameterized Quantile Function (Yang et al., NeurIPS 2019), outside the reference: iqn's
//                 network at taus a fraction proposal layer computes in the step, its own loss kernel and a second
//                 (RMSProp) optimizer launch over the fraction layer (DESIGN.md §15)
//   dueling,      network options of dqn / double_q / prioritized / munchausen, outside the reference: the dueling
//   noisy         network (Wang et al., ICML 2016; DESIGN.md §16) and factorised-noise layers with a mu bias
//                 (Fortunato et al., ICLR 2018; networks.py:137-178 with_bias=True; DESIGN.md §17), alone or together
//
// Gradients flow only through online(s_tm1).  All forward passes of a layer are one grouped
// launch (dz_gemm.cuh); the replay gather is fused into conv1's operand load.
#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

#include "dz_async.cuh"
#include "dz_gemm.cuh"
#include "dz_tc.cuh"
#include "dz_internal.cuh"
#include "dz_umma_net.cuh"

namespace dz {

// The network an agent kind applies: munchausen_iqn and fqf run iqn's network, munchausen dqn's.  Every network-structure
// decision (layout, carving, tensor-core plan, randomness, tau counts, acting) goes through these two predicates; the
// loss launch is the only place that tells a Munchausen kind from the kind whose network it uses.
__host__ __device__ constexpr bool uses_iqn_net(int kind) { return kind == DZ_IQN || kind == DZ_MUNCHAUSEN_IQN || kind == DZ_FQF; }
// fqf (DESIGN.md §15) carries every decision in which it differs from iqn: its taus are proposed in the step from the
// torso features (no draws, no tau inputs, nothing for the randomness calls to generate), its Q-values weight the
// quantiles by the interval widths, and the fraction layer at the end of the blob gets its own optimizer launch.
constexpr bool proposes_fractions(int kind) { return kind == DZ_FQF; }
// iqn's network with taus drawn per step and passed in by the caller (iqn, munchausen_iqn)
constexpr bool draws_taus(int kind) { return uses_iqn_net(kind) && !proposes_fractions(kind); }
__host__ __device__ constexpr bool uses_dqn_net(int kind) { return kind == DZ_DQN || kind == DZ_MUNCHAUSEN; }
// The kind given to the device kernels that branch on the network (q_values_kernel).
constexpr int net_kind(int kind) { return uses_iqn_net(kind) ? DZ_IQN : uses_dqn_net(kind) ? DZ_DQN : kind; }
// The Munchausen kinds: alpha / tau / l0 are validated, and the target network also applies to s_tm1.
constexpr bool is_munchausen(int kind) { return kind == DZ_MUNCHAUSEN || kind == DZ_MUNCHAUSEN_IQN; }
// The kinds whose online network also applies to s_t (double-Q action selection): online(s_tm1) | online(s_t) | target(s_t).
constexpr bool online_applies_to_s_t(int kind) { return kind == DZ_DOUBLE_Q || kind == DZ_PRIORITIZED || kind == DZ_RAINBOW; }
// The kinds that may take the dueling network (DESIGN.md §16) and noisy layers (§17): their losses read one scalar q per
// action.
constexpr bool dueling_allowed(int kind) {
  return kind == DZ_DQN || kind == DZ_DOUBLE_Q || kind == DZ_PRIORITIZED || kind == DZ_MUNCHAUSEN;
}
// After validate(): the network has two 512-wide streams after the torso (rainbow's noisy pair, the dueling network's
// pair), and its layers are noisy (rainbow, noisy networks).  Every decision about the second stream's buffers, plan and
// launches asks the first; every decision about noise asks the second.
inline bool two_streams(const dz_learner_config& c) { return c.kind == DZ_RAINBOW || c.dueling != 0; }
inline bool noisy_net(const dz_learner_config& c) { return c.kind == DZ_RAINBOW || c.noisy != 0; }
// Whether the loss section writes priorities and keeps the running max-seen priority (DESIGN.md §19): prioritized and
// rainbow always, any other kind with the config's prioritized field set.
inline bool writes_priorities(const dz_learner_config& c) {
  return c.kind == DZ_PRIORITIZED || c.kind == DZ_RAINBOW || c.prioritized != 0;
}

// ------------------------------------------------------------------------------------------------
// Parameter layout (canonical names; haiku layouts) — must match oracle/learner_oracle.py:param_shapes
// ------------------------------------------------------------------------------------------------

struct TensorInfo {
  std::string name;
  int64_t shape[4];
  int ndim;
  int64_t offset, count;
};

struct Dims {
  int H, W, C;       // observation
  int h1, w1, h2, w2, h3, w3;
  int feat;          // h3*w3*64
  int out;           // head outputs (family dependent)
};

static Dims make_dims(const dz_learner_config& c) {
  Dims d;
  d.H = c.obs_h; d.W = c.obs_w; d.C = c.obs_c;
  d.h1 = conv_out(d.H, 8, 4); d.w1 = conv_out(d.W, 8, 4);
  d.h2 = conv_out(d.h1, 4, 2); d.w2 = conv_out(d.w1, 4, 2);
  d.h3 = conv_out(d.h2, 3, 1); d.w3 = conv_out(d.w2, 3, 1);
  d.feat = d.h3 * d.w3 * 64;
  switch (c.kind) {
    case DZ_C51: d.out = c.num_actions * c.num_atoms; break;
    case DZ_QRDQN: d.out = c.num_quantiles * c.num_actions; break;
    case DZ_RAINBOW: d.out = c.num_actions * c.num_atoms; break;
    default: d.out = c.num_actions;
  }
  return d;
}

// The layers after the torso of every network but IQN's (which has stream 0 only, with plain layers): one or two
// streams (two: the advantage stream s = 0, then the value stream), each a 3136 -> 512 layer and a head, plain or noisy.
// Rainbow's streams are noisy with GEMM heads; the dueling network's head is one kernel over both streams.
struct FcNet {
  int ns;               // streams
  bool noisy;           // factorised-noise layers: mu and sigma tensors, noise vectors, dual GEMMs
  bool dueling_head;    // the head is dueling_head_fwd/bwd_kernel (or its noisy variant); else a grouped GEMM per stream
  int64_t out[2];       // each stream's head width: d.out; the value stream's num_atoms for rainbow, 1 for dueling
  bool head_mu_bias;    // the head has a mu bias (rainbow's has none: with_bias=False)
  bool shared_bias;     // head/b has shape {1} (plain double_q / prioritized)
};

static FcNet fc_net(const dz_learner_config& c, const Dims& d) {
  const bool rb = c.kind == DZ_RAINBOW;
  FcNet f;
  f.ns = two_streams(c) ? 2 : 1;
  f.noisy = noisy_net(c);
  f.dueling_head = f.ns == 2 && !rb;
  f.out[0] = d.out;
  f.out[1] = f.ns == 2 ? (rb ? c.num_atoms : 1) : 0;
  f.head_mu_bias = !rb;
  f.shared_bias = f.ns == 1 && !f.noisy && (c.kind == DZ_DOUBLE_Q || c.kind == DZ_PRIORITIZED);
  return f;
}

// Offsets into a parameter blob of every tensor the step's launches address; -1 where the agent kind has no such tensor.
// Stream s as in FcNet.  Layer 1 is the 512-wide layer, layer 2 the head; w / b are plain or mu, sw / sb noisy sigma.
struct ParamOffsets {
  int64_t conv_w[3], conv_b[3];
  int64_t w1[2], b1[2], sw1[2], sb1[2];
  int64_t w2[2], b2[2], sw2[2], sb2[2];
  int64_t embed_w, embed_b;
  int64_t frac_w, frac_b;   // fqf's fraction layer; frac_w is also where the fraction tail of the blob begins
  int64_t fc_begin;   // first offset after the conv tensors
};

struct Layout {
  std::vector<TensorInfo> t;
  int64_t total = 0;
  int64_t add(const std::string& name, std::initializer_list<int64_t> shape) {
    TensorInfo ti;
    ti.name = name;
    ti.ndim = (int)shape.size();
    ti.count = 1;
    int i = 0;
    for (auto s : shape) { ti.shape[i++] = s; ti.count *= s; }
    for (; i < 4; ++i) ti.shape[i] = 1;
    ti.offset = total;
    total += (ti.count + 3) / 4 * 4;  // keep every tensor 16-byte aligned for float4 loads
    t.push_back(ti);
    return ti.offset;
  }
};

// The parameter layout of cfg's network, and in *po (when given) the offset of every tensor the step addresses.  After
// the conv tensors: iqn's embedding, the layers of FcNet stream by stream (advantage stream first, so that stream index
// s means the same in rainbow and the dueling network), then fqf's fraction layer.  A plain layer is w, b; a noisy one
// (DESIGN.md §17) mu/w, mu/b, sigma/w, sigma/b.  One stream names its layers fc1 / head, two streams adv1 / adv2 and
// val1 / val2.
static Layout make_layout(const dz_learner_config& c, ParamOffsets* po = nullptr) {
  Layout L;
  ParamOffsets o;
  const Dims d = make_dims(c);
  const FcNet f = fc_net(c, d);
  o.conv_w[0] = L.add("conv1/w", {8, 8, d.C, 32}); o.conv_b[0] = L.add("conv1/b", {32});
  o.conv_w[1] = L.add("conv2/w", {4, 4, 32, 64});  o.conv_b[1] = L.add("conv2/b", {64});
  o.conv_w[2] = L.add("conv3/w", {3, 3, 64, 64});  o.conv_b[2] = L.add("conv3/b", {64});
  for (int s = 0; s < 2; ++s) {
    o.w1[s] = o.b1[s] = o.sw1[s] = o.sb1[s] = -1;
    o.w2[s] = o.b2[s] = o.sw2[s] = o.sb2[s] = -1;
  }
  o.embed_w = o.embed_b = -1;
  o.frac_w = o.frac_b = -1;
  if (uses_iqn_net(c.kind)) { o.embed_w = L.add("embed/w", {c.latent_dim, d.feat}); o.embed_b = L.add("embed/b", {d.feat}); }
  const char* streams[2] = {"adv", "val"};
  for (int s = 0; s < f.ns; ++s)
    for (int layer = 1; layer <= 2; ++layer) {
      const std::string p = f.ns == 2 ? streams[s] + std::to_string(layer) : layer == 1 ? "fc1" : "head";
      const bool head = layer == 2;
      const int64_t n_in = head ? 512 : d.feat, n_out = head ? f.out[s] : 512;
      int64_t* w = head ? o.w2 : o.w1;
      int64_t* b = head ? o.b2 : o.b1;
      if (!f.noisy) {
        w[s] = L.add(p + "/w", {n_in, n_out});
        b[s] = L.add(p + "/b", {head && f.shared_bias ? 1 : n_out});
        continue;
      }
      w[s] = L.add(p + "/mu/w", {n_in, n_out});
      if (!head || f.head_mu_bias) b[s] = L.add(p + "/mu/b", {n_out});
      (head ? o.sw2 : o.sw1)[s] = L.add(p + "/sigma/w", {n_in, n_out});
      (head ? o.sb2 : o.sb1)[s] = L.add(p + "/sigma/b", {n_out});
    }
  // fqf: the fraction proposal layer, last, so that it is one contiguous tail of the blob for its optimizer launch
  if (proposes_fractions(c.kind)) {
    o.frac_w = L.add("fraction/w", {d.feat, c.num_fractions}); o.frac_b = L.add("fraction/b", {c.num_fractions});
  }
  o.fc_begin = uses_iqn_net(c.kind) ? o.embed_w : o.w1[0];
  if (po) *po = o;
  return L;
}

struct Bump {
  char* base;
  int64_t used = 0;
  template <typename T> T* take(int64_t n) {
    int64_t bytes = (n * (int64_t)sizeof(T) + 255) / 256 * 256;
    T* p = base ? reinterpret_cast<T*>(base + used) : nullptr;
    used += bytes;
    return p;
  }
};

// ---- Munchausen DQN per-example arithmetic (DESIGN.md §13), shared by loss_munchausen_kernel and its host twin
// dz_test_munchausen_example.  Each softmax over the target network's A action values enters through two reductions,
// v = max_a qbar(s, a) and S = sum_a exp((qbar(s, a) - v) / tau), which the kernel forms with warp shuffles and the
// host twin with the same xor butterfly over an array.  tau log pi(a|s) = qbar(s, a) - v - tau log S, and the bootstrap
// sum_a pi(a|s_t) (qbar(s_t, a) - tau log pi(a|s_t)) equals v_t + tau log S_t for every a; that form is evaluated: it
// needs no third reduction and has no cancellation.  Explicit fmaf keeps the host and device roundings the same.
constexpr int kMunchausenMaxActions = 18;

inline bool munchausen_params_ok(float alpha, float tau, float l0) {
  return std::isfinite(alpha) && std::isfinite(tau) && std::isfinite(l0) && tau > 0.f && alpha >= 0.f && l0 <= 0.f;
}

__host__ __device__ inline float munchausen_exp(float qbar, float v, float tau) { return expf((qbar - v) / tau); }

struct MunchausenTarget { float target, bonus; };

// alpha clip(tau log pi(a_tm1 | s_tm1), l0, 0)
__host__ __device__ inline float munchausen_bonus(float qbar_tm1_a, float v_tm1, float s_tm1, float alpha, float tau, float l0) {
  const float tau_log_pi = fmaf(-tau, logf(s_tm1), qbar_tm1_a - v_tm1);     // tau log pi(a_tm1 | s_tm1)
  return alpha * fminf(fmaxf(tau_log_pi, l0), 0.f);
}

__host__ __device__ inline MunchausenTarget munchausen_target(float r, float disc, float qbar_tm1_a, float v_tm1, float s_tm1,
                                                              float v_t, float s_t, float alpha, float tau, float l0) {
  const float bonus = munchausen_bonus(qbar_tm1_a, v_tm1, s_tm1, alpha, tau, l0);
  const float boot = fmaf(tau, logf(s_t), v_t);
  return MunchausenTarget{fmaf(disc, boot, r + bonus), bonus};
}

// ---- Munchausen-IQN per-example target arithmetic (DESIGN.md §14), shared by loss_munchausen_iqn_kernel and its host
// twin dz_test_munchausen_iqn_example.  qbar(s, a) is the mean of the target network's quantile samples of that pass,
// summed in row order; the softmax reductions are the warp's (the host twin's butterfly), as for munchausen above.
// The bootstrap of sample j is sum_a pi(a|s_t) (zbar_j(s_t, a) + h(a)) with h(a) = v + tau log S - qbar(a) =
// -tau log pi(a|s_t) >= 0, evaluated as sum_a pi zbar_j + E with the entropy term E = sum_a pi h a sum of non-negative
// terms: no cancellation at large qbar (sum pi qbar - tau logsumexp would cancel).
__host__ __device__ inline float miqn_mean(const float* z, int rows, int A, int a) {
  float s = 0.f;
  for (int j = 0; j < rows; ++j) s += z[(long long)j * A + a];
  return s / (float)rows;
}

__host__ __device__ inline float miqn_h(float qbar, float v, float s, float tau) { return fmaf(tau, logf(s), v - qbar); }

// y_j = r + bonus + disc (sum_a pi(a) zbar_j(a) + E); rb = r + bonus
__host__ __device__ inline float miqn_target(const float* zbar_j, const float* pi, int A, float rb, float disc, float ent) {
  float s = 0.f;
  for (int a = 0; a < A; ++a) s = fmaf(pi[a], zbar_j[a], s);
  return fmaf(disc, s + ent, rb);
}

// ---- FQF per-example fraction arithmetic (DESIGN.md §15), shared by fraction_forward_kernel / loss_fqf_kernel and
// their host twin dz_test_fqf_example.  Every sum runs serially in index order, so the host and the device add in the
// same order, and the result of example e does not depend on how many examples a launch holds.
constexpr int kFqfMaxFractions = 128;   // pass 2 holds 2N rows per example: within the 256 rows of the IQN tau limit

// logits [N] -> q = softmax(logits), tau_0 = 0, tau_i = min(sum_{k<i} q_k, 1), tau_N = 1, tau_hat_i = (tau_i +
// tau_{i+1}) / 2 and the interval weights w_i = tau_{i+1} - tau_i.  The float32 prefix sum can round above 1 when the
// last fractions are small; the clamp keeps 0 <= tau_i <= tau_{i+1} <= 1, so w_i >= 0 and tau_i <= tau_hat_i <= tau_{i+1}
// hold exactly.  tau has N + 1 entries; any output may alias nothing else.
__host__ __device__ inline void fqf_fractions(const float* logits, int N, float* q, float* tau, float* tau_hat, float* w) {
  float m = logits[0];
  for (int i = 1; i < N; ++i) m = fmaxf(m, logits[i]);
  float s = 0.f;
  for (int i = 0; i < N; ++i) { q[i] = expf(logits[i] - m); s += q[i]; }
  for (int i = 0; i < N; ++i) q[i] = q[i] / s;
  tau[0] = 0.f;
  for (int i = 1; i < N; ++i) tau[i] = fminf(tau[i - 1] + q[i - 1], 1.f);
  tau[N] = 1.f;
  for (int i = 0; i < N; ++i) {
    tau_hat[i] = (tau[i] + tau[i + 1]) * 0.5f;
    w[i] = tau[i + 1] - tau[i];
  }
}

// The fraction gradient (the paper's Proposition 1) of one example, chained to the logits: with F(tau) =
// Z(s_tm1, a_tm1, tau), dW1/dtau_i = 2 F(tau_i) - F(tau_hat_i) - F(tau_hat_{i-1}) for i = 1..N-1; tau_i = sum_{k<i} q_k
// gives dq_k = sum_{i>k} dW1/dtau_i, and the softmax dlogit_k = q_k (dq_k - sum_j q_j dq_j).  F_tau[i] = F(tau_i)
// (entries 1..N-1 are read), F_hat[i] = F(tau_hat_i); cot = w_b / B scales the result.  dlogits [N] is also the dq scratch.
__host__ __device__ inline void fqf_dlogits(const float* F_tau, const float* F_hat, const float* q, int N, float cot,
                                            float* dlogits) {
  float acc = 0.f;
  dlogits[N - 1] = 0.f;
  for (int k = N - 2; k >= 0; --k) {
    const int i = k + 1;
    acc += (2.f * F_tau[i] - F_hat[i]) - F_hat[i - 1];
    dlogits[k] = acc;
  }
  float dot = 0.f;
  for (int j = 0; j < N; ++j) dot = fmaf(q[j], dlogits[j], dot);
  for (int k = 0; k < N; ++k) dlogits[k] = cot * (q[k] * (dlogits[k] - dot));
}

// Q(s, a) = sum_i w_i Z(s, a, tau_hat_i) over N quantile rows z [N][A]: fqf's selection in the loss and its acting.
__host__ __device__ inline float fqf_weighted_q(const float* z, const float* w, int N, int A, int a) {
  float s = 0.f;
  for (int i = 0; i < N; ++i) s = fmaf(w[i], z[(long long)i * A + a], s);
  return s;
}

// ---- Dueling head per-row arithmetic (DESIGN.md §16), shared by dueling_head_fwd_kernel / dueling_head_bwd_kernel and
// their host twin dz_test_dueling_example.  Both sums run serially in action order; at A = 1 the mean is adv itself, so
// q = v and dadv = 0 exactly.
constexpr int kDuelingMaxActions = 64;

// q_a = v + (adv_a - m), m = (sum_a adv_a) / A.  q may alias adv.
__host__ __device__ inline void dueling_aggregate(const float* adv, float v, int A, float* q) {
  float s = 0.f;
  for (int a = 0; a < A; ++a) s += adv[a];
  const float m = s / (float)A;
  for (int a = 0; a < A; ++a) q[a] = v + (adv[a] - m);
}

// The aggregation's transpose: dadv_a = dq_a - (sum_a dq_a) / A; returns dval = sum_a dq_a.  dadv may alias dq.
__host__ __device__ inline float dueling_transpose(const float* dq, int A, float* dadv) {
  float s = 0.f;
  for (int a = 0; a < A; ++a) s += dq[a];
  const float m = s / (float)A;
  for (int a = 0; a < A; ++a) dadv[a] = dq[a] - m;
  return s;
}

// ---- CQL(H) per-example arithmetic (DESIGN.md §20), shared by every loss kernel's cql variant and its host twin
// dz_test_cql_example.  From the online network's expected values q [A] on s_tm1: R = logsumexp_a q_a - q_{a_tm1} with
// the max subtracted, evaluated as (m - q_{a_tm1}) + log S, two non-negative terms, so R >= 0 holds in fp32 too; and
// g_a = cot (softmax(q)_a - [a = a_tm1]), the gradient of cot R wrt q_a (cot = alpha w_b / B).  Every sum runs serially
// in action order, so example b's bits do not depend on B.  q and g may live in global or shared memory; g may not
// alias q.  Returns R.
struct CqlArgs {
  float alpha;          // > 0 in the cql variant of each loss kernel (the off variant reads nothing here)
  float* regularizer;   // [B] R_b, or NULL
};

__host__ __device__ inline float cql_example(const float* q, int A, int at, float cot, float* g) {
  float m = q[0];
  for (int a = 1; a < A; ++a) m = fmaxf(m, q[a]);
  float s = 0.f;
  for (int a = 0; a < A; ++a) s += expf(q[a] - m);
  for (int a = 0; a < A; ++a) g[a] = cot * (expf(q[a] - m) / s - (a == at ? 1.0f : 0.0f));
  return (m - q[at]) + logf(s);
}

// ---- random-shift augmentation (DESIGN.md §18): the largest pad, and the shared-memory stage of random_shift_kernel,
// which holds the source rows of one band of output rows (84x84x4 and 84x92x4 observations: one band)
constexpr int kShiftMaxPad = 16;
constexpr int kShiftStageBytes = 32768;

static int validate(const dz_learner_config& c) {
  if (c.kind < 0 || c.kind > DZ_FQF) return fail(DZ_EINVAL, "unknown agent kind");
  if (c.dueling != 0 && c.dueling != 1) return fail(DZ_EINVAL, "dueling must be 0 or 1");
  if (c.dueling && !dueling_allowed(c.kind))
    return fail(DZ_EINVAL, "dueling: only dqn, double_q, prioritized and munchausen take the dueling network");
  if (c.noisy != 0 && c.noisy != 1) return fail(DZ_EINVAL, "noisy must be 0 or 1");
  if (c.prioritized != 0 && c.prioritized != 1) return fail(DZ_EINVAL, "prioritized must be 0 or 1");
  if (!std::isfinite(c.cql_alpha) || c.cql_alpha < 0.f) return fail(DZ_EINVAL, "cql_alpha must be finite and >= 0");
  if (c.noisy && c.kind == DZ_RAINBOW) return fail(DZ_EINVAL, "noisy: rainbow's network is noisy already");
  if (c.noisy && !dueling_allowed(c.kind))
    return fail(DZ_EINVAL, "noisy: only dqn, double_q, prioritized and munchausen take noisy layers");
  if (is_munchausen(c.kind) && !munchausen_params_ok(c.munchausen_alpha, c.entropy_temperature, c.log_policy_clip))
    return fail(DZ_EINVAL, "munchausen needs finite alpha >= 0, entropy_temperature > 0 and log_policy_clip <= 0");
  if (is_munchausen(c.kind) && c.num_actions > kMunchausenMaxActions)
    return fail(DZ_EINVAL, "munchausen: num_actions must be in [1,18] (one warp lane per action)");
  // The loss hyperparameters of every kind: the kernels take them as given, so a NaN or a sign error would train on
  // silently wrong targets (a support of -vmax..vmax turned inside out, a negative clip range or Huber width).
  if (!std::isfinite(c.vmax) || !(c.vmax > 0.f)) return fail(DZ_EINVAL, "vmax must be finite and > 0");
  if (!std::isfinite(c.huber_param) || c.huber_param < 0.f) return fail(DZ_EINVAL, "huber_param must be finite and >= 0");
  if (!std::isfinite(c.grad_error_bound) || c.grad_error_bound < 0.f)
    return fail(DZ_EINVAL, "grad_error_bound must be finite and >= 0");
  if (c.batch <= 0 || c.batch > 1024) return fail(DZ_EINVAL, "batch must be in [1,1024]");
  if (c.obs_c != 4) return fail(DZ_EINVAL, "obs_c must be 4 (stacked frames; conv1 reads uchar4 pixels)");
  if (c.obs_w % 4) return fail(DZ_EINVAL, "obs_w must be a multiple of 4");
  if (c.obs_h < 36 || c.obs_w < 36) return fail(DZ_EINVAL, "observation too small for the Nature-CNN torso");
  if (c.random_shift_pad < 0 || c.random_shift_pad > kShiftMaxPad) return fail(DZ_EINVAL, "random_shift_pad must be in [0,16]");
  if (c.random_shift_pad >= std::min(c.obs_h, c.obs_w)) return fail(DZ_EINVAL, "random_shift_pad must be less than min(obs_h, obs_w)");
  if (c.random_shift_pad && (int64_t)c.obs_w * c.obs_c > kShiftStageBytes)
    return fail(DZ_EINVAL, "random_shift_pad: an observation row (obs_w * obs_c bytes) must be at most 32768 bytes");
  if (c.num_actions <= 0 || c.num_actions > 64) return fail(DZ_EINVAL, "num_actions must be in [1,64]");
  if ((c.kind == DZ_C51 || c.kind == DZ_RAINBOW) && (c.num_atoms < 2 || c.num_atoms > 128)) return fail(DZ_EINVAL, "num_atoms must be in [2,128]");
  if (c.kind == DZ_QRDQN && (c.num_quantiles < 1 || c.num_quantiles > 256)) return fail(DZ_EINVAL, "num_quantiles must be in [1,256]");
  if (proposes_fractions(c.kind)) {
    if (c.num_fractions < 2 || c.num_fractions > kFqfMaxFractions) return fail(DZ_EINVAL, "fqf: num_fractions must be in [2,128]");
    if (!std::isfinite(c.fraction_learning_rate) || c.fraction_learning_rate < 0.f)
      return fail(DZ_EINVAL, "fqf: fraction_learning_rate must be finite and >= 0");
    if (!std::isfinite(c.fraction_opt_eps) || !(c.fraction_opt_eps > 0.f))
      return fail(DZ_EINVAL, "fqf: fraction_opt_eps must be finite and > 0");
    if (!(c.fraction_rms_decay >= 0.f && c.fraction_rms_decay < 1.f))
      return fail(DZ_EINVAL, "fqf: fraction_rms_decay must be in [0,1)");
  }
  if (uses_iqn_net(c.kind)) {
    if (c.latent_dim <= 0 || c.latent_dim % 16) return fail(DZ_EINVAL, "latent_dim must be a positive multiple of 16");
  }
  if (draws_taus(c.kind)) {
    int mx = c.tau_samples_s_tm1 > c.tau_samples_s_t ? c.tau_samples_s_tm1 : c.tau_samples_s_t;
    mx = mx > c.tau_samples_policy ? mx : c.tau_samples_policy;
    if (c.tau_samples_s_tm1 <= 0 || c.tau_samples_s_t <= 0 || c.tau_samples_policy <= 0 || mx > 256)
      return fail(DZ_EINVAL, "tau sample counts must be in [1,256]");
  }
  return DZ_OK;
}

}  // namespace dz

using namespace dz;

// ------------------------------------------------------------------------------------------------
// Small kernels
// ------------------------------------------------------------------------------------------------

namespace {

struct FinishNN {  // split-K partials of an NN problem -> bias / noisy combine / relu
  const float* partial; int splits; long long stride; int M, N; int dual;
  const float* bias; const float* bias2; const float* c_scale; int relu; int bias_shared; float* out;
};
struct FinishNNBatch { FinishNN f[kMaxProblems]; int n; };

// ROW_NOISE: row m of a noisy layer carries its own noise apply, its eps_out at c_scale + m * c_ld.
template <bool ROW_NOISE>
__device__ __forceinline__ void finish_nn_body(const FinishNNBatch& b, long long c_ld) {
  const FinishNN& f = b.f[blockIdx.y];
  long long total = (long long)f.M * f.N;
  if ((f.N & 3) == 0 && ((reinterpret_cast<uintptr_t>(f.partial) | reinterpret_cast<uintptr_t>(f.out) | (uintptr_t)(f.stride * 4)) & 15) == 0) {
    // 16-byte path (every layer except the odd-width heads): same per-element order of additions
    const long long total4 = total >> 2;
    for (long long i4 = blockIdx.x * (long long)blockDim.x + threadIdx.x; i4 < total4; i4 += (long long)gridDim.x * blockDim.x) {
      const long long i = i4 << 2;
      const int n = (int)(i % f.N);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int k = 0; k < f.splits; ++k) {
        const float4 x = *reinterpret_cast<const float4*>(f.partial + k * f.stride + i);
        v.x += x.x; v.y += x.y; v.z += x.z; v.w += x.w;
      }
      if (f.bias) {
        if (f.bias_shared) { const float s = f.bias[0]; v.x += s; v.y += s; v.z += s; v.w += s; }
        else { v.x += f.bias[n]; v.y += f.bias[n + 1]; v.z += f.bias[n + 2]; v.w += f.bias[n + 3]; }
      }
      if (f.dual && f.bias2) {
        const float* eo = ROW_NOISE ? f.c_scale + (i / f.N) * c_ld : f.c_scale;
        v.x = fmaf(f.bias2[n], eo[n], v.x); v.y = fmaf(f.bias2[n + 1], eo[n + 1], v.y);
        v.z = fmaf(f.bias2[n + 2], eo[n + 2], v.z); v.w = fmaf(f.bias2[n + 3], eo[n + 3], v.w);
      }
      if (f.relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
      *reinterpret_cast<float4*>(f.out + i) = v;
    }
    return;
  }
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int n = (int)(i % f.N);
    float v = 0.f;
    for (int k = 0; k < f.splits; ++k) v += f.partial[k * f.stride + i];
    if (f.bias) v += f.bias_shared ? f.bias[0] : f.bias[n];
    if (f.dual && f.bias2) {   // sigma bias of the noisy layer
      const float* eo = ROW_NOISE ? f.c_scale + (i / f.N) * c_ld : f.c_scale;
      v = fmaf(f.bias2[n], eo[n], v);
    }
    if (f.relu) v = fmaxf(v, 0.f);
    f.out[i] = v;
  }
}

__global__ void __launch_bounds__(256) finish_nn_kernel(const __grid_constant__ FinishNNBatch b) {
  dz::pdl_enter();
  finish_nn_body<false>(b, 0);
}

__global__ void __launch_bounds__(256) finish_nn_rownoise_kernel(const __grid_constant__ FinishNNBatch b, long long c_ld) {
  dz::pdl_enter();
  finish_nn_body<true>(b, c_ld);
}

struct FinishTN {  // split partials [Kext][N] of a TN problem -> weight / bias gradients
  const float* partial; int splits; long long stride; int K, N;
  float* C; float* C2; float* Cb; float* Cb2; const float* a_scale; const float* c_scale;
};
struct FinishTNBatch { FinishTN f[kMaxProblems]; int n; };

__global__ void __launch_bounds__(256) finish_tn_kernel(const __grid_constant__ FinishTNBatch b) {
  dz::pdl_enter();
  const FinishTN& f = b.f[blockIdx.y];
  int Kext = f.K + ((f.Cb || f.Cb2) ? 1 : 0);
  long long total = (long long)Kext * f.N;
  if ((f.N & 3) == 0 && !f.C2 && !f.Cb2 && f.C &&
      ((reinterpret_cast<uintptr_t>(f.partial) | reinterpret_cast<uintptr_t>(f.C) | reinterpret_cast<uintptr_t>(f.Cb) | (uintptr_t)(f.stride * 4)) & 15) == 0) {
    const long long total4 = total >> 2;
    for (long long i4 = blockIdx.x * (long long)blockDim.x + threadIdx.x; i4 < total4; i4 += (long long)gridDim.x * blockDim.x) {
      const long long i = i4 << 2;
      const int k = (int)(i / f.N), n = (int)(i % f.N);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int s = 0; s < f.splits; ++s) {
        const float4 x = *reinterpret_cast<const float4*>(f.partial + s * f.stride + i);
        v.x += x.x; v.y += x.y; v.z += x.z; v.w += x.w;
      }
      if (k < f.K) *reinterpret_cast<float4*>(f.C + i) = v;
      else if (f.Cb) *reinterpret_cast<float4*>(f.Cb + n) = v;
    }
    return;
  }
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int k = (int)(i / f.N), n = (int)(i % f.N);
    float v = 0.f;
    for (int s = 0; s < f.splits; ++s) v += f.partial[s * f.stride + i];
    if (k < f.K) {
      if (f.C) f.C[i] = v;
      if (f.C2) f.C2[i] = v * f.a_scale[k] * f.c_scale[n];
    } else {
      if (f.Cb) f.Cb[n] = v;
      if (f.Cb2) f.Cb2[n] = v * f.c_scale[n];
    }
  }
}

struct FinishNT {  // split partials [M][K] (+ dual second half) of up to two NT problems -> summed, masked output
  const float* partial[2]; const float* a_scale[2]; int nsrc; int splits; long long stride; int M, K; int dual;
  const float* mask; float* out;
  float* out_hi; float* out_lo;   // optional: the tf32 hi/lo pair the tensor-core kernels read (saves a separate split launch)
};
struct FinishNTBatch { FinishNT f[2]; };   // blockIdx.y selects the job

__global__ void __launch_bounds__(256) finish_nt_kernel(const __grid_constant__ FinishNTBatch fb) {
  dz::pdl_enter();
  const FinishNT& f = fb.f[blockIdx.y];
  long long total = (long long)f.M * f.K;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    float v = 0.f;
    for (int q = 0; q < f.nsrc; ++q) {
      float a = 0.f;
      for (int s = 0; s < f.splits; ++s) a += f.partial[q][s * f.stride + i];
      v += a;
    }
    if (f.mask && !(f.mask[i] > 0.f)) v = 0.f;
    f.out[i] = v;
    if (f.out_hi) {
      float h, l;
      tc::split_tf32(v, h, l);
      f.out_hi[i] = h;
      f.out_lo[i] = l;
    }
  }
}

// col2im for the conv input gradient: dX[b,y,x,c] = sum over kernel taps of dcol, times ReLU mask.
__global__ void __launch_bounds__(256) col2im_kernel(const float* __restrict__ dcol, const float* __restrict__ act,
                                                     float* __restrict__ dx, int nimg, int H, int W, int Cin, int KH, int KW,
                                                     int S, int OH, int OW) {
  dz::pdl_enter();
  long long total = (long long)nimg * H * W * Cin;
  const int K = KH * KW * Cin;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % Cin);
    long long t = i / Cin;
    int x = (int)(t % W); t /= W;
    int y = (int)(t % H);
    int b = (int)(t / H);
    float v = 0.f;
    if (act[i] > 0.f) {
      for (int kh = 0; kh < KH; ++kh) {
        int yy = y - kh;
        if (yy < 0 || yy % S) continue;
        int oy = yy / S;
        if (oy >= OH) continue;
        for (int kw = 0; kw < KW; ++kw) {
          int xx = x - kw;
          if (xx < 0 || xx % S) continue;
          int ox = xx / S;
          if (ox >= OW) continue;
          v += dcol[((long long)(b * OH + oy) * OW + ox) * K + (kh * KW + kw) * Cin + c];
        }
      }
    }
    dx[i] = v;
  }
}

__global__ void sum_to_scalar_kernel(const float* __restrict__ v, int n, float* out) {
  dz::pdl_enter();
  __shared__ float s[32];
  float acc = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) acc += v[i];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    acc = threadIdx.x < (blockDim.x >> 5) ? s[threadIdx.x] : 0.f;
    acc = warp_sum(acc);
    if (threadIdx.x == 0) out[0] = acc;
  }
}

// ---- IQN helpers -------------------------------------------------------------------------------

// IQN value head at training size (networks.py:285-287): out[m, a] = sum_k h1[m, k] W[k, a] + b[a] with
// M = batch * tau_samples rows (thousands), K = 512 and only num_actions (<= 18) columns.  A tiled GEMM wastes its
// N tile here; instead one warp owns one row: coalesced float4 reads of the row, W^T resident in shared memory,
// A warp reductions.  Up to three applies (blockIdx.y) per launch.
constexpr int kSkinnyMaxN = 18;
struct SkinnyHead { const float* A[3]; const float* W[3]; const float* bias[3]; float* out[3]; int M[3]; int n; };

__global__ void __launch_bounds__(256) iqn_head_fwd_kernel(const __grid_constant__ SkinnyHead h, int N) {
  dz::pdl_enter();
  constexpr int K = 512;
  __shared__ __align__(16) float Ws[kSkinnyMaxN * K];
  const int q = blockIdx.y;
  const float* __restrict__ W = h.W[q];
  for (int i = threadIdx.x; i < K * N; i += 256) {      // W is [K][N]: transpose into Ws[n][k]
    int k = i / N, n = i - k * N;
    Ws[n * K + k] = W[i];
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int m = blockIdx.x * 8 + warp; m < h.M[q]; m += gridDim.x * 8) {
    const float4* a4 = reinterpret_cast<const float4*>(h.A[q] + (long long)m * K);
    float4 a[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) a[i] = a4[lane + 32 * i];
    float mine = 0.f;
    for (int n = 0; n < N; ++n) {
      const float4* w4 = reinterpret_cast<const float4*>(Ws + n * K);
      float acc = 0.f;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float4 w = w4[lane + 32 * i];
        acc = fmaf(a[i].x, w.x, acc); acc = fmaf(a[i].y, w.y, acc); acc = fmaf(a[i].z, w.z, acc); acc = fmaf(a[i].w, w.w, acc);
      }
      acc = warp_sum(acc);
      if (lane == n) mine = acc;
    }
    if (lane < N) h.out[q][(long long)m * N + lane] = mine + h.bias[q][lane];
  }
}

// Input gradient of the same head: dh1[m, k] = [h1 > 0] * sum_a dout[m, a] W[k, a]  (one thread = 4 consecutive k).
__global__ void __launch_bounds__(256) iqn_head_dgrad_kernel(const float* __restrict__ dout, const float* __restrict__ W,
                                                             const float* __restrict__ h1, float* __restrict__ dh1, int M, int N) {
  dz::pdl_enter();
  constexpr int K = 512;
  __shared__ float Ws[K * kSkinnyMaxN];
  for (int i = threadIdx.x; i < K * N; i += 256) Ws[i] = W[i];
  __syncthreads();
  const long long total = (long long)M * (K / 4);
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int m = (int)(i >> 7), k = (int)(i & 127) * 4;
    float d[kSkinnyMaxN];
    for (int n = 0; n < N; ++n) d[n] = dout[(long long)m * N + n];
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int n = 0; n < N; ++n) {
      v.x = fmaf(d[n], Ws[(k + 0) * N + n], v.x);
      v.y = fmaf(d[n], Ws[(k + 1) * N + n], v.y);
      v.z = fmaf(d[n], Ws[(k + 2) * N + n], v.z);
      v.w = fmaf(d[n], Ws[(k + 3) * N + n], v.w);
    }
    const float4 h = *reinterpret_cast<const float4*>(h1 + (long long)m * K + k);
    v.x = h.x > 0.f ? v.x : 0.f; v.y = h.y > 0.f ? v.y : 0.f; v.z = h.z > 0.f ? v.z : 0.f; v.w = h.w > 0.f ? v.w : 0.f;
    *reinterpret_cast<float4*>(dh1 + (long long)m * K + k) = v;
  }
}

// cos(pi * i * tau), i = 1..latent; the product is formed in float32 as in networks.py:277-278.
__global__ void iqn_cos_kernel(const float* __restrict__ taus, float* __restrict__ out, long long rows, int latent) {
  dz::pdl_enter();
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= rows * latent) return;
  int j = (int)(i % latent);
  float pim = __fmul_rn((float)(j + 1), 3.14159274101257324f);
  out[i] = cosf(__fmul_rn(pim, taus[i / latent]));
}

// dE = dHI * F * (E > 0) in place; dF[b,k] = sum_n dHI[b,n,k] * E[b,n,k]; dfeat masked by act3 > 0.
__global__ void __launch_bounds__(256) iqn_hadamard_bwd_kernel(float* __restrict__ dHI, const float* __restrict__ E,
                                                               const float* __restrict__ F, float* __restrict__ dfeat,
                                                               int B, int N, int D) {
  dz::pdl_enter();
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)B * D) return;
  int b = (int)(i / D), k = (int)(i % D);
  float f = F[i], acc = 0.f;
  for (int n = 0; n < N; ++n) {
    long long j = ((long long)b * N + n) * D + k;
    float g = dHI[j], e = E[j];
    acc += g * e;
    dHI[j] = e > 0.f ? g * f : 0.f;
  }
  dfeat[i] = f > 0.f ? acc : 0.f;  // F is the post-ReLU conv3 output: mask for the conv3 pre-activation
}

// Packed variant for the tensor-core path: same math, but dE is written ONLY as the hi/lo TF32 tile images of the
// transposed operand (rows k, reduction m = b*N + n; layout: pk_index) that the embedding weight-gradient GEMM
// consumes.  One block = one sample b x 64 features; requires N == 64 and D % 64 == 0.
__global__ void __launch_bounds__(256) iqn_hadamard_bwd_packed_kernel(const float* __restrict__ dHI, const float* __restrict__ E,
                                                                      const float* __restrict__ F, float* __restrict__ dfeat,
                                                                      float* __restrict__ img_hi, float* __restrict__ img_lo,
                                                                      int rg_total, int D) {
  dz::pdl_enter();
  constexpr int N = 64;
  __shared__ float tile[64][65];
  __shared__ float red[16][64];
  const int b = blockIdx.y, k0 = blockIdx.x * 64, tid = threadIdx.x;
  const int a = tid >> 4, k4 = (tid & 15) * 4;
  const float4 f = *reinterpret_cast<const float4*>(F + (long long)b * D + k0 + k4);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int n = a + 16 * q;
    const long long j = ((long long)b * N + n) * D + k0 + k4;
    const float4 g = *reinterpret_cast<const float4*>(dHI + j);
    const float4 e = *reinterpret_cast<const float4*>(E + j);
    acc.x = fmaf(g.x, e.x, acc.x); acc.y = fmaf(g.y, e.y, acc.y); acc.z = fmaf(g.z, e.z, acc.z); acc.w = fmaf(g.w, e.w, acc.w);
    tile[n][k4 + 0] = e.x > 0.f ? g.x * f.x : 0.f;
    tile[n][k4 + 1] = e.y > 0.f ? g.y * f.y : 0.f;
    tile[n][k4 + 2] = e.z > 0.f ? g.z * f.z : 0.f;
    tile[n][k4 + 3] = e.w > 0.f ? g.w * f.w : 0.f;
  }
  red[a][k4 + 0] = acc.x; red[a][k4 + 1] = acc.y; red[a][k4 + 2] = acc.z; red[a][k4 + 3] = acc.w;
  __syncthreads();
  if (tid < 64) {
    float sum = 0.f;
#pragma unroll
    for (int r = 0; r < 16; ++r) sum += red[r][tid];
    const long long i = (long long)b * D + k0 + tid;
    dfeat[i] = F[i] > 0.f ? sum : 0.f;   // F is the post-ReLU conv3 output: mask for the conv3 pre-activation
  }
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int id = tid + q * 256;
    const int r = id & 7, c = (id >> 3) & 3, rg = (id >> 5) & 7, kb = id >> 8;
    const int k = k0 + rg * 8 + r, ml = kb * 16 + c * 4;
    float4 x = make_float4(tile[ml][rg * 8 + r], tile[ml + 1][rg * 8 + r], tile[ml + 2][rg * 8 + r], tile[ml + 3][rg * 8 + r]);
    float4 h, l;
    tc::split_tf32(x, h, l);
    const long long off = pk_index(k, b * N + ml, rg_total);
    *reinterpret_cast<float4*>(img_hi + off) = h;
    *reinterpret_cast<float4*>(img_lo + off) = l;
  }
}

// ---- randomness --------------------------------------------------------------------------------

__device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1,
                                              uint32_t out[4]) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

// kind 0: U[0,1) (IQN taus); kind 1: sign(n)*sqrt|n|, n ~ TruncNormal(-2,2) (networks.py:142-144).
__global__ void randomness_kernel(float* __restrict__ out, long long n, uint64_t seed, const int64_t* counters, int kind,
                                  uint32_t stream_id) {
  dz::pdl_enter();
  long long i4 = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i4 * 4 >= n) return;
  uint64_t ctr = (uint64_t)counters[1];
  uint32_t r[4];
  philox4x32_10((uint32_t)i4, (uint32_t)(i4 >> 32), (uint32_t)ctr, (uint32_t)(ctr >> 32) ^ (stream_id << 24), (uint32_t)seed,
                (uint32_t)(seed >> 32), r);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    long long i = i4 * 4 + j;
    if (i >= n) break;
    float u = (float)(r[j] >> 8) * (1.0f / 16777216.0f);  // [0,1)
    if (kind == 0) {
      out[i] = u;
    } else {
      const float lo = -0.95449973610364158f;  // erf(-2/sqrt(2))
      float v = lo + (-2.0f * lo) * ((float)(r[j] >> 8) + 0.5f) * (1.0f / 16777216.0f);
      float x = 1.41421356237f * erfinvf(v);
      x = fminf(fmaxf(x, -2.0f), 2.0f);
      out[i] = copysignf(sqrtf(fabsf(x)), x);
    }
  }
}

__global__ void bump_counter_kernel(int64_t* counters, int which) {
  dz::pdl_enter(); counters[which] += 1; }

// ---- random-shift augmentation (DESIGN.md §18) ---------------------------------------------------

// The shifts of one update: example b takes the Philox block at counter (b, 0, ctr low, ctr high ^ (3 << 24)) and its
// words w give (dy0, dx0, dy1, dx1) = floor(w (2p + 1) / 2^32).  Reads the counter, does not advance it.
__global__ void shift_draw_kernel(int32_t* __restrict__ out, int B, int pad, uint64_t seed, const int64_t* counters) {
  dz::pdl_enter();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const uint64_t ctr = (uint64_t)counters[1];
  uint32_t r[4];
  philox4x32_10((uint32_t)b, 0u, (uint32_t)ctr, (uint32_t)(ctr >> 32) ^ (3u << 24), (uint32_t)seed, (uint32_t)(seed >> 32), r);
  const uint32_t span = 2u * (uint32_t)pad + 1u;
#pragma unroll
  for (int j = 0; j < 4; ++j) out[4 * b + j] = (int32_t)__umulhi(r[j], span);
}

struct ShiftArgs {
  const uint8_t* const* src[2];   // [B] row tables of s_tm1 and s_t, [H][W][C] each
  const int32_t* shifts;          // [B][4]: (dy0, dx0, dy1, dx1)
  uint8_t* out;                   // [B][2][stride]
  long long stride;               // a multiple of 16, >= H * W * C
  const uint8_t** rows[2];        // when set, rows[i][b] <- the shifted observation (the tables the torso then reads)
  int H, W, C, pad;
};

constexpr int kShiftThreads = 256;

// One CTA per (observation i = s_tm1 | s_t, example b): out[y][x][c] = in[clamp(y + dy - p)][clamp(x + dx - p)][c].  The
// source rows of a band of output rows are contiguous: they are staged through shared memory with 16-byte loads, and
// each output 16-byte word is gathered from the stage in 32-bit pixel words (C % 4 == 0) and stored whole.
__global__ void __launch_bounds__(kShiftThreads) random_shift_kernel(const __grid_constant__ ShiftArgs a) {
  __shared__ uint4 stage[kShiftStageBytes / 16];
  dz::pdl_enter();
  const int i = blockIdx.x, b = blockIdx.y, p = a.pad;
  const int dy = min(max(a.shifts[4 * b + 2 * i], 0), 2 * p) - p;
  const int dx = min(max(a.shifts[4 * b + 2 * i + 1], 0), 2 * p) - p;
  const int rw = a.W * a.C / 16;   // 16-byte words per row
  const int cw = a.C / 4;          // 32-bit words per pixel
  const uint4* src = reinterpret_cast<const uint4*>(a.src[i][b]);
  uint4* dst = reinterpret_cast<uint4*>(a.out + ((long long)b * 2 + i) * a.stride);
  if (a.rows[i] != nullptr && threadIdx.x == 0) a.rows[i][b] = reinterpret_cast<const uint8_t*>(dst);
  const uint32_t* st = reinterpret_cast<const uint32_t*>(stage);
  const int band = kShiftStageBytes / 16 / rw;
  for (int y0 = 0; y0 < a.H; y0 += band) {
    const int y1 = min(a.H, y0 + band);
    // clamp is monotone and 1-Lipschitz: the band's source rows s0..s1 are at most y1 - y0
    const int s0 = min(max(y0 + dy, 0), a.H - 1), s1 = min(max(y1 - 1 + dy, 0), a.H - 1);
    const int n = (s1 - s0 + 1) * rw;
    const uint4* from = src + (long long)s0 * rw;
#pragma unroll 4
    for (int k = threadIdx.x; k < n; k += kShiftThreads) stage[k] = __ldg(from + k);
    __syncthreads();
    const int m = (y1 - y0) * rw;
    for (int k = threadIdx.x; k < m; k += kShiftThreads) {
      const int yy = k / rw, kw = k - yy * rw;
      const uint32_t* row = st + (min(max(y0 + yy + dy, 0), a.H - 1) - s0) * rw * 4;
      uint32_t v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int wd = 4 * kw + j;
        const int px = cw == 1 ? wd : wd / cw;
        v[j] = row[min(max(px + dx, 0), a.W - 1) * cw + (wd - px * cw)];
      }
      dst[(long long)(y0 + yy) * rw + kw] = make_uint4(v[0], v[1], v[2], v[3]);
    }
    __syncthreads();
  }
  const long long obs16 = (long long)a.H * rw, tail16 = a.stride / 16 - obs16;   // the row's stride padding is zero
  for (long long k = threadIdx.x; k < tail16; k += kShiftThreads) dst[obs16 + k] = make_uint4(0u, 0u, 0u, 0u);
}

// ---- losses ------------------------------------------------------------------------------------

struct LossArgs {
  int kind, B, A, atoms, N, Ksel, Nt;  // N: #src quantiles (s_tm1), Ksel: selector samples, Nt: target samples
  const float* out0; const float* out1; const float* out2;       // head outputs of pass 0 / 1 / 2 (see learner)
  const float* adv0; const float* val0; const float* adv1; const float* val1; const float* adv2; const float* val2;  // rainbow
  const int32_t* a; const float* r; const float* disc; const float* w; const float* taus0;
  float vmax, bound, kappa;
  float* dout; float* dadv; float* dval;      // gradients wrt pass-0 head outputs
  float* per_example; float* priorities; float* loss_terms;  // loss_terms[b] = w_b * loss_b
};

__device__ __forceinline__ float block_sum(float v, float* smem) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) smem[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = threadIdx.x < (blockDim.x >> 5) ? smem[threadIdx.x] : 0.f;
  if (threadIdx.x < 32) t = warp_sum(t);
  if (threadIdx.x == 0) smem[0] = t;
  __syncthreads();
  t = smem[0];
  __syncthreads();
  return t;
}
__device__ __forceinline__ float block_max(float v, float* smem) {
  v = warp_max(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) smem[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = threadIdx.x < (blockDim.x >> 5) ? smem[threadIdx.x] : -INFINITY;
  if (threadIdx.x < 32) t = warp_max(t);
  if (threadIdx.x == 0) smem[0] = t;
  __syncthreads();
  t = smem[0];
  __syncthreads();
  return t;
}

// dqn / double_q / prioritized: rlax.q_learning / double_q_learning, clip_gradient, l2_loss.  kCql (DESIGN.md §20): the
// CQL term on the online head's q-values, its gradient added to dout unclipped.
template <bool kCql>
__global__ void __launch_bounds__(64) loss_q_kernel(LossArgs L, CqlArgs cq) {
  dz::pdl_enter();
  int b = blockIdx.x;
  if (threadIdx.x != 0) return;
  const float* q_tm1 = L.out0 + (long long)b * L.A;
  const float* q_sel = (L.kind == DZ_DQN ? L.out2 : L.out1) + (long long)b * L.A;
  const float* q_tgt = L.out2 + (long long)b * L.A;
  int best = 0;
  for (int a = 1; a < L.A; ++a)
    if (q_sel[a] > q_sel[best]) best = a;
  int at = L.a[b];
  float target = L.r[b] + L.disc[b] * q_tgt[best];
  float td = target - q_tm1[at];
  float w = L.w ? L.w[b] : 1.0f;
  float g = fminf(fmaxf(w * td / (float)L.B, -L.bound), L.bound);  // cotangent reaching clip_gradient
  if constexpr (kCql) {
    float* d = L.dout + (long long)b * L.A;
    const float R = cql_example(q_tm1, L.A, at, cq.alpha * w / (float)L.B, d);
    d[at] -= g;
    L.per_example[b] = td;
    if (L.priorities) L.priorities[b] = fabsf(td);
    if (cq.regularizer) cq.regularizer[b] = R;
    L.loss_terms[b] = w * fmaf(cq.alpha, R, 0.5f * td * td);
  } else {
    for (int a = 0; a < L.A; ++a) L.dout[(long long)b * L.A + a] = (a == at) ? -g : 0.f;
    L.per_example[b] = td;
    if (L.priorities) L.priorities[b] = fabsf(td);                   // prioritized/agent.py:201
    L.loss_terms[b] = w * 0.5f * td * td;
  }
}

// munchausen: one warp per example, lane a holding action a of the target network's passes on s_tm1 (out1) and s_t
// (out2); the target of DESIGN.md §13, then dqn's clip_gradient + l2_loss on td = target - q(s_tm1, a_tm1).  The
// per-example value is the loss 0.5 td^2; the priority is |td|, the dqn family's rule on the soft target.  kCql
// (DESIGN.md §20): lane 0 adds the CQL term on the online head's q-values (out0), its gradient unclipped.
template <bool kCql>
__global__ void __launch_bounds__(128) loss_munchausen_kernel(LossArgs L, float alpha, float tau, float l0, CqlArgs cq) {
  dz::pdl_enter();
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= L.B) return;   // the whole warp leaves together
  const int A = L.A;
  const long long row = (long long)b * A;
  const bool act = lane < A;
  const float qbar_tm1 = act ? L.out1[row + lane] : -INFINITY;
  const float qbar_t = act ? L.out2[row + lane] : -INFINITY;
  const float v_tm1 = warp_max(qbar_tm1), v_t = warp_max(qbar_t);
  const float s_tm1 = warp_sum(act ? munchausen_exp(qbar_tm1, v_tm1, tau) : 0.f);
  const float s_t = warp_sum(act ? munchausen_exp(qbar_t, v_t, tau) : 0.f);
  const int at = L.a[b];
  const float qbar_a = __shfl_sync(0xffffffffu, qbar_tm1, at);
  const MunchausenTarget m = munchausen_target(L.r[b], L.disc[b], qbar_a, v_tm1, s_tm1, v_t, s_t, alpha, tau, l0);
  const float td = m.target - L.out0[row + at];
  const float w = L.w ? L.w[b] : 1.0f;
  const float g = fminf(fmaxf(w * td / (float)L.B, -L.bound), L.bound);   // cotangent reaching clip_gradient
  if constexpr (kCql) {
    if (lane == 0) {
      const float R = cql_example(L.out0 + row, A, at, cq.alpha * w / (float)L.B, L.dout + row);
      L.dout[row + at] -= g;
      const float loss = 0.5f * td * td;
      L.per_example[b] = loss;
      if (L.priorities) L.priorities[b] = fabsf(td);
      if (cq.regularizer) cq.regularizer[b] = R;
      L.loss_terms[b] = w * fmaf(cq.alpha, R, loss);
    }
  } else {
    if (act) L.dout[row + lane] = lane == at ? -g : 0.f;
    if (lane == 0) {
      const float loss = 0.5f * td * td;
      L.per_example[b] = loss;
      if (L.priorities) L.priorities[b] = fabsf(td);
      L.loss_terms[b] = w * loss;
    }
  }
}

// c51 / rainbow: categorical_[double_]q_learning with categorical_l2_project + cross entropy.
// One CTA (4 warps) per example.  Everything the example's loss reads from the three head passes is first staged in
// shared memory; softmaxes then run one warp per (pass, action) with shuffle reductions, so the whole kernel has six
// block barriers.  Dynamic shared memory: categorical_loss_smem().  kCql (DESIGN.md §20): step 1 also takes every
// action's expected value Q_a under the online(s_tm1) pass, step 2 the CQL coefficients of those Q_a, and step 5 chains
// them through dQ_a / dlogit_{a,k} = p_{a,k} (z_k - Q_a) into every action's logits (rainbow: through the aggregation's
// transpose into dadv and dval).
template <bool kCql>
__global__ void __launch_bounds__(128) loss_categorical_staged_kernel(LossArgs L, CqlArgs cq) {
  dz::pdl_enter();
  extern __shared__ float sm[];
  const int b = blockIdx.x, K = L.atoms, A = L.A, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  float* cm_sel = sm;            // [K] mean over actions of the selector-pass advantages (rainbow)
  float* cm_tgt = cm_sel + K;    // [K] same for the target pass
  float* cm_tm1 = cm_tgt + K;    // [K] same for the online(s_tm1) pass
  float* p_tgt = cm_tm1 + K;     // [K]
  float* proj = p_tgt + K;       // [K]
  float* p_tm1 = proj + K;       // [K] softmax(logits_tm1[a_tm1])
  float* qsel = p_tm1 + K;       // [A]
  float* scal = qsel + A;        // [4]: loss, sum(proj)
  float* zs = scal + 4;          // [K] support atoms
  float* st_adv = zs + K;        // [3][A*K] head outputs of this example for pass 0 / 1 / 2
  float* st_val = st_adv + 3 * A * K;   // [3][K] value-stream outputs (rainbow)
  // kCql, after st_val: [A] Q_a of online(s_tm1), [A] max and [A] denominator of each action's softmax of that pass,
  // [A] the CQL gradient wrt Q_a, [1] R (indexed from st_val + 3K inside the kCql blocks)
  const bool rb = L.kind == DZ_RAINBOW;
  // Everything this example's loss reads from the three head passes goes to shared memory in ONE round of coalesced,
  // independent loads; the phases below are then shared-memory arithmetic instead of ~10 dependent global round trips.
  {
    const float* __restrict__ a0 = (rb ? L.adv0 : L.out0) + (long long)b * A * K;
    const float* __restrict__ a1 = (rb ? L.adv1 : L.out2) + (long long)b * A * K;
    const float* __restrict__ a2 = (rb ? L.adv2 : L.out2) + (long long)b * A * K;
    for (int i = tid; i < A * K; i += blockDim.x) {
      const float x0 = a0[i], x1 = a1[i], x2 = a2[i];
      st_adv[i] = x0; st_adv[A * K + i] = x1; st_adv[2 * A * K + i] = x2;
    }
    if (rb) {
      const float* __restrict__ v0 = L.val0 + (long long)b * K;
      const float* __restrict__ v1 = L.val1 + (long long)b * K;
      const float* __restrict__ v2 = L.val2 + (long long)b * K;
      for (int i = tid; i < K; i += blockDim.x) {
        const float x0 = v0[i], x1 = v1[i], x2 = v2[i];
        st_val[i] = x0; st_val[K + i] = x1; st_val[2 * K + i] = x2;
      }
    }
    for (int i = tid; i < K; i += blockDim.x) zs[i] = (float)((double)(-L.vmax) + (double)i * (2.0 * (double)L.vmax / (double)(K - 1)));
  }
  __syncthreads();
  auto support = [&](int i) { return zs[i]; };

  // 0. dueling column means (networks.py:251: mean over the action axis)
  if (rb) {
    for (int k = tid; k < K; k += blockDim.x) {
      float m1 = 0.f, m2 = 0.f, m0 = 0.f;
      for (int a = 0; a < A; ++a) {
        m1 += st_adv[A * K + a * K + k];
        m2 += st_adv[2 * A * K + a * K + k];
        m0 += st_adv[a * K + k];
      }
      cm_sel[k] = m1 / (float)A; cm_tgt[k] = m2 / (float)A; cm_tm1[k] = m0 / (float)A;
    }
  }
  __syncthreads();
  // logit k of (pass, action): pass 0 = online(s_tm1), 1 = selector, 2 = target
  auto logit_of = [&](int pass, int a, int k) -> float {
    if (rb) {
      const float* cm = pass == 0 ? cm_tm1 : (pass == 1 ? cm_sel : cm_tgt);
      return st_val[pass * K + k] + st_adv[pass * A * K + a * K + k] - cm[k];
    }
    return st_adv[(pass == 0 ? 0 : 2) * A * K + a * K + k];   // c51 selects with the target network
  };
  // warp-level softmax of (pass, a): returns this lane's max/denominator; optionally writes probabilities
  auto warp_softmax = [&](int pass, int a, float* probs, float& mx, float& den) {
    float m = -INFINITY;
    for (int k = lane; k < K; k += 32) m = fmaxf(m, logit_of(pass, a, k));
    mx = warp_max(m);
    float s = 0.f;
    for (int k = lane; k < K; k += 32) s += expf(logit_of(pass, a, k) - mx);
    den = warp_sum(s);
    if (probs)
      for (int k = lane; k < K; k += 32) probs[k] = expf(logit_of(pass, a, k) - mx) / den;
  };

  // 1. selector q-values, one warp per action
  for (int a = warp; a < A; a += 4) {
    float mx, den;
    warp_softmax(rb ? 1 : 2, a, nullptr, mx, den);
    float s = 0.f;
    for (int k = lane; k < K; k += 32) s += (expf(logit_of(rb ? 1 : 2, a, k) - mx) / den) * support(k);
    s = warp_sum(s);
    if (lane == 0) qsel[a] = s;
    if constexpr (kCql) {
      warp_softmax(0, a, nullptr, mx, den);
      float s0 = 0.f;
      for (int k = lane; k < K; k += 32) s0 += (expf(logit_of(0, a, k) - mx) / den) * support(k);
      s0 = warp_sum(s0);
      float* cq = st_val + 3 * K;
      if (lane == 0) { cq[a] = s0; cq[A + a] = mx; cq[2 * A + a] = den; }
    }
  }
  __syncthreads();
  int best = 0;
  for (int a = 1; a < A; ++a)
    if (qsel[a] > qsel[best]) best = a;
  const int at = L.a[b];
  // 2. target distribution (warp 0) and softmax of the taken action's online logits (warp 1)
  float mx_tm1 = 0.f, den_tm1 = 1.f;
  if (warp == 0) { float mx, den; warp_softmax(2, best, p_tgt, mx, den); }
  if (warp == 1) {
    warp_softmax(0, at, p_tm1, mx_tm1, den_tm1);
    if (lane == 0) { scal[2] = mx_tm1; scal[3] = den_tm1; }
  }
  if constexpr (kCql) {
    float* q0 = st_val + 3 * K;
    if (tid == 64) q0[4 * A] = cql_example(q0, A, at, cq.alpha * (L.w ? L.w[b] : 1.0f) / (float)L.B, q0 + 3 * A);
  }
  __syncthreads();
  // 3. rlax.categorical_l2_project(r + discount*z, p, z)
  const float r = L.r[b], dsc = L.disc[b];
  const float zmin = support(0), zmax = support(K - 1);
  for (int i = tid; i < K; i += blockDim.x) {
    float zi = support(i);
    float dpos = (i + 1 < K ? support(i + 1) : support(0)) - zi;      // roll(z,-1) - z
    float dneg = zi - (i > 0 ? support(i - 1) : support(K - 1));      // z - roll(z,1)
    dpos = dpos > 0.f ? 1.0f / dpos : 0.f;
    dneg = dneg > 0.f ? 1.0f / dneg : 0.f;
    float acc = 0.f;
    for (int j = 0; j < K; ++j) {
      float zp = fminf(fmaxf(r + dsc * support(j), zmin), zmax);
      float delta = zp - zi;
      float dhat = delta >= 0.f ? delta * dpos : -(delta * dneg);
      acc += fminf(fmaxf(1.0f - dhat, 0.f), 1.0f) * p_tgt[j];
    }
    proj[i] = acc;
  }
  __syncthreads();
  // 4. cross entropy with log_softmax(logits_tm1[a_tm1]) (warp 0)
  if (warp == 0) {
    const float mx = scal[2], logden = logf(scal[3]);
    float ls = 0.f, ps = 0.f;
    for (int k = lane; k < K; k += 32) {
      ls += proj[k] * (logit_of(0, at, k) - mx - logden);
      ps += proj[k];
    }
    ls = warp_sum(ls); ps = warp_sum(ps);
    if (lane == 0) { scal[0] = -ls; scal[1] = ps; }
  }
  __syncthreads();
  const float loss = scal[0], psum = scal[1];
  const float w = L.w ? L.w[b] : 1.0f;
  const float cot = w / (float)L.B;
  // 5. gradient wrt the pass-0 head outputs
  if constexpr (kCql) {
    const float* q0 = st_val + 3 * K;
    // the CQL gradient wrt logit k of action a (pass 0)
    auto cql_dlogit = [&](int a, int k) {
      const float p0 = expf(logit_of(0, a, k) - q0[A + a]) / q0[2 * A + a];
      return q0[3 * A + a] * (p0 * (support(k) - q0[a]));
    };
    if (rb) {
      for (int k = tid; k < K; k += blockDim.x) {
        const float dl = cot * (p_tm1[k] * psum - proj[k]);
        float s = 0.f;
        for (int a = 0; a < A; ++a) s += (a == at ? dl : 0.f) + cql_dlogit(a, k);
        L.dval[(long long)b * K + k] = s;
        const float m = s / (float)A;
        for (int a = 0; a < A; ++a) L.dadv[((long long)b * A + a) * K + k] = ((a == at ? dl : 0.f) + cql_dlogit(a, k)) - m;
      }
    } else {
      for (int i = tid; i < A * K; i += blockDim.x) {
        int a = i / K, k = i - a * K;
        L.dout[(long long)b * A * K + i] = ((a == at) ? cot * (p_tm1[k] * psum - proj[k]) : 0.f) + cql_dlogit(a, k);
      }
    }
    if (tid == 0) {
      L.per_example[b] = loss;
      if (L.priorities) L.priorities[b] = fminf(fmaxf(fabsf(loss), 0.f), 100.f);
      if (cq.regularizer) cq.regularizer[b] = q0[4 * A];
      L.loss_terms[b] = w * fmaf(cq.alpha, q0[4 * A], loss);
    }
    return;
  }
  if (rb) {
    for (int k = tid; k < K; k += blockDim.x) {
      float dl = cot * (p_tm1[k] * psum - proj[k]);
      L.dval[(long long)b * K + k] = dl;
      for (int a = 0; a < A; ++a)
        L.dadv[((long long)b * A + a) * K + k] = dl * ((a == at ? 1.0f : 0.0f) - 1.0f / (float)A);
    }
  } else {
    for (int i = tid; i < A * K; i += blockDim.x) {
      int a = i / K, k = i - a * K;
      L.dout[(long long)b * A * K + i] = (a == at) ? cot * (p_tm1[k] * psum - proj[k]) : 0.f;
    }
  }
  if (tid == 0) {
    L.per_example[b] = loss;
    if (L.priorities) L.priorities[b] = fminf(fmaxf(fabsf(loss), 0.f), 100.f);  // rainbow/agent.py:194
    L.loss_terms[b] = w * loss;
  }
}

// 6K + A + 4 floats of working arrays, K support atoms, and the staged [3][A*K] head outputs and [3][K] value outputs.
// The largest configuration validate() accepts (A = 64, K = 128) needs 103,696 bytes, more than the default 48 KB.
// cql_alpha > 0 adds 4A + 1 floats (kCql's Q_a, softmax maxima and denominators, coefficients and R).
size_t categorical_loss_smem(const dz_learner_config& c) {
  const size_t A = c.num_actions, K = c.num_atoms;
  return (6 * K + A + 4 + K + 3 * A * K + 3 * K + (c.cql_alpha > 0.f ? 4 * A + 1 : 0)) * sizeof(float);
}

// rlax.quantile_regression_loss of example b's N source quantiles src (at taus tau) against its Nt targets tgt, all in
// shared memory, and the gradient wrt the pass-0 head outputs in IQN's layout (nonzero at a_tm1 only): the tail of
// loss_quantile_kernel, which keeps its own inline copy so that its code generation stays as it was.  kCql (DESIGN.md
// §20): dout also takes the CQL gradient coef[a] * dQ_a / dZ_{i,a}, with the row weight roww[i] (fqf) or 1/N (the mean),
// and the loss term alpha r[0]; cql_quantile_head prepares coef and r.
template <bool kCql = false>
__device__ __forceinline__ void quantile_huber_tail(const LossArgs& L, int b, int at, int N, int Nt, const float* tgt,
                                                    const float* src, const float* tau, float* red,
                                                    const CqlArgs* cq = nullptr, const float* coef = nullptr,
                                                    const float* roww = nullptr, const float* r = nullptr) {
  const int A = L.A, tid = threadIdx.x;
  const float kappa = L.kappa;
  const float w = L.w ? L.w[b] : 1.0f;
  const float cot = w / (float)L.B;
  float total = 0.f;
  for (int i = tid; i < N; i += blockDim.x) {
    float acc = 0.f, gacc = 0.f;
    for (int j = 0; j < Nt; ++j) {
      float delta = tgt[j] - src[i];
      float wt = fabsf(tau[i] - (delta < 0.f ? 1.0f : 0.0f));
      float ad = fabsf(delta);
      float l, dl;
      if (kappa > 0.f) {
        float q = fminf(ad, kappa);
        l = 0.5f * q * q + kappa * (ad - q);
        dl = fminf(fmaxf(delta, -kappa), kappa);
      } else {
        l = ad;
        dl = delta > 0.f ? 1.0f : (delta < 0.f ? -1.0f : 0.0f);
      }
      acc += wt * l;
      gacc += wt * dl;
    }
    total += acc / (float)Nt;
    float g = -cot * gacc / (float)Nt;  // d loss / d src_i  (delta = target - src)
    if constexpr (kCql) {
      const float rw = roww ? roww[i] : 1.0f / (float)N;
      for (int a = 0; a < A; ++a) L.dout[((long long)b * N + i) * A + a] = ((a == at) ? g : 0.f) + coef[a] * rw;
    } else {
      for (int a = 0; a < A; ++a) L.dout[((long long)b * N + i) * A + a] = (a == at) ? g : 0.f;
    }
  }
  total = block_sum(total, red);
  if (tid == 0) {
    L.per_example[b] = total;
    if (L.priorities) L.priorities[b] = fminf(fmaxf(fabsf(total), 0.f), 100.f);   // rainbow's rule, DESIGN.md §19
    if constexpr (kCql) {
      if (cq->regularizer) cq->regularizer[b] = r[0];
      L.loss_terms[b] = w * fmaf(cq->alpha, r[0], total);
    } else {
      L.loss_terms[b] = w * total;
    }
  }
}

// kCql's head of the quantile kernels (DESIGN.md §20): Q_a of online(s_tm1)'s N rows z0 [N][A], their mean or, with
// roww, sum_i roww[i] z0[i][a] (fqf), one thread per action in row order; then R to r[0] and the coefficients coef [A]
// (cql_example).  q, coef and r are shared memory; every thread of the CTA calls it.
__device__ __forceinline__ void cql_quantile_head(const float* z0, int N, int A, const float* roww, int at, float cot,
                                                  float* q, float* coef, float* r) {
  const int tid = threadIdx.x;
  if (tid < A) q[tid] = roww ? fqf_weighted_q(z0, roww, N, A, tid) : miqn_mean(z0, N, A, tid);
  __syncthreads();
  if (tid == 0) r[0] = cql_example(q, A, at, cot, coef);
  __syncthreads();
}

// qrdqn / iqn: rlax.quantile_q_learning with quantile_regression_loss (Huber kappa).
// Layouts: qrdqn out[b, q*A + a] (networks.py:308), iqn out[(b*N + n)*A + a] (networks.py:286-287).  kCql (DESIGN.md
// §20): Q_a is the mean of the pass-0 quantiles, and the tail is quantile_huber_tail's cql variant.
template <bool kCql>
__global__ void __launch_bounds__(256) loss_quantile_kernel(LossArgs L, CqlArgs cq) {
  dz::pdl_enter();
  extern __shared__ float sm[];
  const int b = blockIdx.x, A = L.A, tid = threadIdx.x;
  const bool iqn = L.kind == DZ_IQN;
  const int N = L.N, Ks = L.Ksel, Nt = L.Nt;
  float* red = sm;            // [32]
  float* qsel = sm + 32;      // [A]
  float* tgt = qsel + A;      // [Nt]
  float* src = tgt + Nt;      // [N]
  float* tau = src + N;       // [N]
  // selector: mean over samples of the selector distribution (qrdqn: the target dist itself)
  const float* sel = iqn ? L.out1 + (long long)b * Ks * A : L.out2 + (long long)b * Nt * A;
  const int nsel = iqn ? Ks : Nt;
  for (int a = 0; a < A; ++a) {
    float s = 0.f;
    for (int j = tid; j < nsel; j += blockDim.x) s += sel[(long long)j * A + a];
    s = block_sum(s, red);
    if (tid == 0) qsel[a] = s / (float)nsel;
    __syncthreads();
  }
  int best = 0;
  for (int a = 1; a < A; ++a)
    if (qsel[a] > qsel[best]) best = a;
  const int at = L.a[b];
  const float r = L.r[b], dsc = L.disc[b];
  const float* dist_t = L.out2 + (long long)b * Nt * A;
  const float* dist_s = L.out0 + (long long)b * N * A;
  for (int j = tid; j < Nt; j += blockDim.x) tgt[j] = r + dsc * dist_t[(long long)j * A + best];
  for (int i = tid; i < N; i += blockDim.x) {
    src[i] = dist_s[(long long)i * A + at];
    tau[i] = iqn ? L.taus0[(long long)b * N + i] : ((float)i + 0.5f) / (float)N;  // qrdqn/run_atari.py:137
  }
  __syncthreads();
  if constexpr (kCql) {
    float* cq_q = tau + N;        // [A]
    float* cq_coef = cq_q + A;    // [A]
    float* cq_r = cq_coef + A;    // [1]
    cql_quantile_head(dist_s, N, A, nullptr, at, cq.alpha * (L.w ? L.w[b] : 1.0f) / (float)L.B, cq_q, cq_coef, cq_r);
    quantile_huber_tail<true>(L, b, at, N, Nt, tgt, src, tau, red, &cq, cq_coef, nullptr, cq_r);
    return;
  }
  const float kappa = L.kappa;
  const float w = L.w ? L.w[b] : 1.0f;
  const float cot = w / (float)L.B;
  float total = 0.f;
  for (int i = tid; i < N; i += blockDim.x) {
    float acc = 0.f, gacc = 0.f;
    for (int j = 0; j < Nt; ++j) {
      float delta = tgt[j] - src[i];
      float wt = fabsf(tau[i] - (delta < 0.f ? 1.0f : 0.0f));
      float ad = fabsf(delta);
      float l, dl;
      if (kappa > 0.f) {
        float q = fminf(ad, kappa);
        l = 0.5f * q * q + kappa * (ad - q);
        dl = fminf(fmaxf(delta, -kappa), kappa);
      } else {
        l = ad;
        dl = delta > 0.f ? 1.0f : (delta < 0.f ? -1.0f : 0.0f);
      }
      acc += wt * l;
      gacc += wt * dl;
    }
    total += acc / (float)Nt;
    float g = -cot * gacc / (float)Nt;  // d loss / d src_i  (delta = target - src)
    for (int a = 0; a < A; ++a) L.dout[((long long)b * N + i) * A + a] = (a == at) ? g : 0.f;
  }
  total = block_sum(total, red);
  if (tid == 0) {
    L.per_example[b] = total;
    if (L.priorities) L.priorities[b] = fminf(fmaxf(fabsf(total), 0.f), 100.f);   // rainbow's rule, DESIGN.md §19
    L.loss_terms[b] = w * total;
  }
}

// munchausen_iqn (DESIGN.md §14): one CTA per example.  (1) qbar of target(s_tm1) over its K policy samples (out1) and
// of target(s_t) over its N' samples (out2), one thread per (pass, action), in row order; (2) one warp, lane a holding
// action a: both softmaxes, the log-policy bonus and the entropy term E = sum_a pi(a|s_t) h(a); (3) the N' targets
// y_j = r + bonus + disc (sum_a pi(a|s_t) zbar_j(s_t, a) + E); (4) IQN's quantile-Huber term of online(s_tm1)'s N
// samples at a_tm1 against them and (5) dout in IQN's layout (quantile_huber_tail).  The per-example value is the loss.
// kCql (DESIGN.md §20): Q_a is the mean of online(s_tm1)'s N samples, and the tail is quantile_huber_tail's cql variant.
template <bool kCql>
__global__ void __launch_bounds__(256) loss_munchausen_iqn_kernel(LossArgs L, float alpha, float tau_e, float l0, CqlArgs cq) {
  dz::pdl_enter();
  extern __shared__ float sm[];
  const int b = blockIdx.x, A = L.A, tid = threadIdx.x;
  const int N = L.N, K = L.Ksel, Nt = L.Nt;
  float* red = sm;            // [32]
  float* qbar = sm + 32;      // [2][A]: s_tm1, s_t
  float* pi = qbar + 2 * A;   // [A]: pi(a|s_t)
  float* scal = pi + A;       // [2]: bonus, E
  float* tgt = scal + 2;      // [Nt]
  float* src = tgt + Nt;      // [N]
  float* tau = src + N;       // [N]
  const float* zbar_tm1 = L.out1 + (long long)b * K * A;
  const float* zbar_t = L.out2 + (long long)b * Nt * A;
  if (tid < 2 * A) {
    const bool t = tid >= A;
    qbar[tid] = miqn_mean(t ? zbar_t : zbar_tm1, t ? Nt : K, A, t ? tid - A : tid);
  }
  __syncthreads();
  const int at = L.a[b];
  if (tid < 32) {
    const bool act = tid < A;
    const float q1 = act ? qbar[tid] : -INFINITY, q2 = act ? qbar[A + tid] : -INFINITY;
    const float v1 = warp_max(q1), v2 = warp_max(q2);
    const float s1 = warp_sum(act ? munchausen_exp(q1, v1, tau_e) : 0.f);
    const float e2 = act ? munchausen_exp(q2, v2, tau_e) : 0.f;
    const float s2 = warp_sum(e2);
    const float p2 = e2 / s2;
    const float ent = warp_sum(act ? p2 * miqn_h(q2, v2, s2, tau_e) : 0.f);
    if (act) pi[tid] = p2;
    if (tid == 0) { scal[0] = munchausen_bonus(qbar[at], v1, s1, alpha, tau_e, l0); scal[1] = ent; }
  }
  __syncthreads();
  const float rb = L.r[b] + scal[0], dsc = L.disc[b], ent = scal[1];
  for (int j = tid; j < Nt; j += blockDim.x) tgt[j] = miqn_target(zbar_t + (long long)j * A, pi, A, rb, dsc, ent);
  const float* dist_s = L.out0 + (long long)b * N * A;
  for (int i = tid; i < N; i += blockDim.x) {
    src[i] = dist_s[(long long)i * A + at];
    tau[i] = L.taus0[(long long)b * N + i];
  }
  __syncthreads();
  if constexpr (kCql) {
    float* cq_q = tau + N;        // [A]
    float* cq_coef = cq_q + A;    // [A]
    float* cq_r = cq_coef + A;    // [1]
    cql_quantile_head(dist_s, N, A, nullptr, at, cq.alpha * (L.w ? L.w[b] : 1.0f) / (float)L.B, cq_q, cq_coef, cq_r);
    quantile_huber_tail<true>(L, b, at, N, Nt, tgt, src, tau, red, &cq, cq_coef, nullptr, cq_r);
  } else {
    quantile_huber_tail(L, b, at, N, Nt, tgt, src, tau, red);
  }
}

// cql_alpha > 0 adds 2A + 1 floats (the cql variant's Q_a, coefficients and R).
size_t munchausen_iqn_loss_smem(const dz_learner_config& c) {
  return (32 + 3 * (size_t)c.num_actions + 2 + c.tau_samples_s_t + 2 * (size_t)c.tau_samples_s_tm1 +
          (c.cql_alpha > 0.f ? 2 * (size_t)c.num_actions + 1 : 0)) * sizeof(float);
}

// ---- fqf (DESIGN.md §15) ------------------------------------------------------------------------

// The fraction proposal layer on the torso features of E examples and up to two applications (blockIdx.y), one CTA per
// (example, application): logits = feat . W + b with W = fraction/w [D][N], then fqf_fractions.  Each of the 8 warps
// takes every 8th feature row in order and the partials are added in warp order, so example e's bits do not depend on
// E.  Every output may be NULL.  The learner's two pass inputs are written here too: pass1 = tau_1..tau_N of
// application 0 (online(s_tm1), no gradient; row N-1 is tau_N = 1, which no loss term reads) and pass2 = [tau_hat of
// application 1 | tau_hat of application 0] (target(s_t): the selection rows, then the target rows).
struct FracArgs {
  const float* feat[2];               // [E][D] torso features of each application
  const float* W; const float* bias;  // the online blob's fraction layer
  int N, D;
  float* tau[2];       // [E][N + 1]
  float* tau_hat[2];   // [E][N]
  float* w[2];         // [E][N]
  float* q[2];         // [E][N]
  float* pass1;        // [E][N]
  float* pass2;        // [E][2N]
};

__global__ void __launch_bounds__(256) fraction_forward_kernel(const __grid_constant__ FracArgs f) {
  dz::pdl_enter();
  constexpr int kMax = kFqfMaxFractions;
  __shared__ float part[8][kMax];
  __shared__ float logits[kMax], q[kMax], tau[kMax + 1], hat[kMax], w[kMax];
  const int e = blockIdx.x, app = blockIdx.y, N = f.N, D = f.D, tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const float* __restrict__ x = f.feat[app] + (long long)e * D;
  for (int c0 = 0; c0 < N; c0 += 32) {
    const int col = c0 + lane;
    if (col >= N) continue;
    float acc = 0.f;
#pragma unroll 4
    for (int k = warp; k < D; k += 8) acc = fmaf(x[k], f.W[(long long)k * N + col], acc);
    part[warp][col] = acc;
  }
  __syncthreads();
  if (tid < N) {
    float s = 0.f;
#pragma unroll
    for (int r = 0; r < 8; ++r) s += part[r][tid];
    logits[tid] = s + f.bias[tid];
  }
  __syncthreads();
  if (tid == 0) fqf_fractions(logits, N, q, tau, hat, w);
  __syncthreads();
  const long long row = (long long)e * N;
  for (int i = tid; i <= N; i += blockDim.x) {
    if (f.tau[app]) f.tau[app][(long long)e * (N + 1) + i] = tau[i];
    if (i == N) continue;
    if (f.tau_hat[app]) f.tau_hat[app][row + i] = hat[i];
    if (f.w[app]) f.w[app][row + i] = w[i];
    if (f.q[app]) f.q[app][row + i] = q[i];
    if (app == 0 && f.pass1) f.pass1[row + i] = tau[i + 1];
    if (f.pass2) f.pass2[2 * row + (app == 0 ? N : 0) + i] = hat[i];
  }
}

struct FqfLossArgs {
  const float* w_t;     // [B][N] interval weights of the proposal on target(s_t)'s features (application 1)
  const float* q_tm1;   // [B][N] softmax of the proposal on online(s_tm1)'s features (application 0)
  float* dlogits;       // [B][N] gradient of the weighted fraction loss wrt the fraction logits of application 0
};

// fqf: one CTA per example.  out0 = online(s_tm1) at tau_hat (N rows), out1 = online(s_tm1) at tau_1..tau_N (N rows, no
// gradient), out2 = target(s_t) at [tau_hat' | tau_hat] (2N rows); taus0 = tau_hat.  (1) the selection a* = argmax_a
// sum_i w'_i Zbar(s_t, a, tau_hat'_i), one thread per action, first maximum; (2) the targets y_j = r + discount
// Zbar(s_t, a*, tau_hat_j); (3) the fraction gradient at a_tm1 chained to dlogits (fqf_dlogits, thread 0); (4) IQN's
// quantile-Huber term of online(s_tm1)'s N samples at a_tm1 against the targets and dout in IQN's layout
// (quantile_huber_tail).  The per-example value, and the priority's source, is the quantile loss.  kCql (DESIGN.md §20):
// Q_a = sum_i w_i Z(s_tm1, tau_hat_i, a) with the interval weights w_i of s_tm1's proposal, formed from q_tm1 by
// fqf_fractions' recurrence (the bits fraction_forward_kernel wrote) and held constant, and the tail is
// quantile_huber_tail's cql variant.
template <bool kCql>
__global__ void __launch_bounds__(256) loss_fqf_kernel(LossArgs L, FqfLossArgs f, CqlArgs cq) {
  dz::pdl_enter();
  extern __shared__ float sm[];
  const int b = blockIdx.x, A = L.A, N = L.N, tid = threadIdx.x;
  float* red = sm;           // [32]
  float* qsel = red + 32;    // [A]
  float* tgt = qsel + A;     // [N]
  float* src = tgt + N;      // [N] F(tau_hat_i)
  float* tau = src + N;      // [N] tau_hat_i
  float* ftau = tau + N;     // [N] F(tau_i), i >= 1
  float* q = ftau + N;       // [N]
  float* dl = q + N;         // [N]
  const float* zsel = L.out2 + (long long)b * 2 * N * A;
  if (tid < A) qsel[tid] = fqf_weighted_q(zsel, f.w_t + (long long)b * N, N, A, tid);
  const int at = L.a[b];
  const float* z0 = L.out0 + (long long)b * N * A;
  const float* z1 = L.out1 + (long long)b * N * A;
  for (int i = tid; i < N; i += blockDim.x) {
    src[i] = z0[(long long)i * A + at];
    tau[i] = L.taus0[(long long)b * N + i];
    ftau[i] = i > 0 ? z1[(long long)(i - 1) * A + at] : 0.f;
    q[i] = f.q_tm1[(long long)b * N + i];
  }
  __syncthreads();
  int best = 0;
  for (int a = 1; a < A; ++a)
    if (qsel[a] > qsel[best]) best = a;
  const float r = L.r[b], dsc = L.disc[b];
  const float* ztgt = zsel + (long long)N * A;
  for (int j = tid; j < N; j += blockDim.x) tgt[j] = r + dsc * ztgt[(long long)j * A + best];
  if (tid == 0) fqf_dlogits(ftau, src, q, N, (L.w ? L.w[b] : 1.0f) / (float)L.B, dl);
  __syncthreads();
  for (int k = tid; k < N; k += blockDim.x) f.dlogits[(long long)b * N + k] = dl[k];
  if constexpr (kCql) {
    float* cw = dl + N;           // [N] interval weights of s_tm1's proposal
    float* cq_q = cw + N;         // [A]
    float* cq_coef = cq_q + A;    // [A]
    float* cq_r = cq_coef + A;    // [1]
    if (tid == 0) {
      float t = 0.f;              // tau_i; tau_N = 1
      for (int i = 0; i < N; ++i) {
        const float next = i + 1 < N ? fminf(t + q[i], 1.f) : 1.f;
        cw[i] = next - t;
        t = next;
      }
    }
    __syncthreads();
    cql_quantile_head(z0, N, A, cw, at, cq.alpha * (L.w ? L.w[b] : 1.0f) / (float)L.B, cq_q, cq_coef, cq_r);
    quantile_huber_tail<true>(L, b, at, N, N, tgt, src, tau, red, &cq, cq_coef, cw, cq_r);
  } else {
    quantile_huber_tail(L, b, at, N, N, tgt, src, tau, red);
  }
}

// cql_alpha > 0 adds N + 2A + 1 floats (the cql variant's interval weights, Q_a, coefficients and R).
size_t fqf_loss_smem(const dz_learner_config& c) {
  return (32 + (size_t)c.num_actions + 6 * (size_t)c.num_fractions +
          (c.cql_alpha > 0.f ? (size_t)c.num_fractions + 2 * (size_t)c.num_actions + 1 : 0)) * sizeof(float);
}

__global__ void loss_mean_kernel(const float* __restrict__ terms, int B, float* loss, float* max_seen, const float* priorities) {
  dz::pdl_enter();
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    float s = 0.f;
    for (int b = 0; b < B; ++b) s += terms[b];
    loss[0] = s / (float)B;
    if (max_seen && priorities) {
      float m = max_seen[0];
      for (int b = 0; b < B; ++b) m = fmaxf(m, priorities[b]);
      max_seen[0] = m;  // rainbow/agent.py:196-197
    }
  }
}

// q_values of one head pass (select_action): c51/rainbow expectation, qr/iqn mean, dqn identity.
// blockIdx.x = environment stream (batched acting); one block for the single-observation call.
__global__ void __launch_bounds__(128) q_values_kernel(int kind, int A, int atoms, int nq, float vmax, const float* out,
                                                       const float* adv, const float* val, float* q) {
  dz::pdl_enter();
  extern __shared__ float sm[];
  float* red = sm;
  float* logit = sm + 32;
  const int tid = threadIdx.x;
  {
    const long long e = blockIdx.x;
    const long long per_img = (kind == DZ_C51 || kind == DZ_RAINBOW) ? (long long)A * atoms
                              : ((kind == DZ_QRDQN || kind == DZ_IQN) ? (long long)nq * A : (long long)A);
    out += e * per_img; adv += e * per_img; if (val) val += e * atoms; q += e * A;
  }
  for (int a = 0; a < A; ++a) {
    float res;
    if (kind == DZ_C51 || kind == DZ_RAINBOW) {
      const int K = atoms;
      for (int k = tid; k < K; k += blockDim.x) {
        if (kind == DZ_RAINBOW) {
          float m = 0.f;
          for (int aa = 0; aa < A; ++aa) m += adv[aa * K + k];
          logit[k] = val[k] + adv[a * K + k] - m / (float)A;
        } else {
          logit[k] = out[a * K + k];
        }
      }
      __syncthreads();
      float m = -INFINITY;
      for (int k = tid; k < K; k += blockDim.x) m = fmaxf(m, logit[k]);
      m = block_max(m, red);
      float s = 0.f, e = 0.f;
      for (int k = tid; k < K; k += blockDim.x) {
        float p = expf(logit[k] - m);
        s += p;
        e += p * (float)((double)(-vmax) + (double)k * (2.0 * (double)vmax / (double)(K - 1)));
      }
      s = block_sum(s, red);
      e = block_sum(e, red);
      res = e / s;
    } else if (kind == DZ_QRDQN || kind == DZ_IQN) {
      float s = 0.f;
      for (int j = tid; j < nq; j += blockDim.x) s += out[(long long)j * A + a];
      res = block_sum(s, red) / (float)nq;
    } else {
      res = out[a];
    }
    if (tid == 0) q[a] = res;
    __syncthreads();
  }
}

// fqf's q-values of one N-row head pass per observation (blockIdx.x): Q(s, a) = sum_i w_i Z(s, a, tau_hat_i), the
// weighting of the loss kernel's selection (fqf_weighted_q); out [E][N][A], w [E][N].
__global__ void __launch_bounds__(64) q_values_fqf_kernel(int A, int N, const float* __restrict__ out, const float* __restrict__ w,
                                                          float* __restrict__ q) {
  dz::pdl_enter();
  const long long e = blockIdx.x;
  for (int a = threadIdx.x; a < A; a += blockDim.x) q[e * A + a] = fqf_weighted_q(out + e * N * A, w + e * N, N, A, a);
}

// ---- optimizer ---------------------------------------------------------------------------------

// Sum of squares -> per-block partials; the last block to finish adds them in a fixed order
// (deterministic), publishes the global norm and bumps the optimizer step count.
// sumsq_only: norm_out[0] receives the SUM OF SQUARES of the range (the split global norm: the optimizer adds the
// conv-gradient partials written by the weight-gradient finish kernels and takes the root), user_norm is not written.
__global__ void __launch_bounds__(256) grad_norm_kernel(const float* __restrict__ g, long long n, float* partials,
                                                        unsigned int* ticket, float* norm_out, int64_t* counters, float* user_norm,
                                                        int sumsq_only) {
  dz::pdl_enter();
  __shared__ float s[32];
  __shared__ bool last;
  float acc = 0.f;
  const long long n4 = n >> 2;   // the blob is padded to a multiple of 4 floats
  const float4* g4 = reinterpret_cast<const float4*>(g);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 v = g4[i];
    acc = fmaf(v.x, v.x, acc); acc = fmaf(v.y, v.y, acc); acc = fmaf(v.z, v.z, acc); acc = fmaf(v.w, v.w, acc);
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < (blockDim.x >> 5); ++i) t += s[i];
    partials[blockIdx.x] = t;
    __threadfence();
    unsigned int done = atomicAdd(ticket, 1u);
    last = (done == gridDim.x - 1);
  }
  __syncthreads();
  if (last) {   // fixed-order tree over the per-block partials: deterministic whatever block finishes last
    __threadfence();
    float t = 0.f;
    for (unsigned int i = threadIdx.x; i < gridDim.x; i += blockDim.x) t += ((volatile float*)partials)[i];
    t = warp_sum(t);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = t;
    __syncthreads();
    if (threadIdx.x == 0) {
      float tot = 0.f;
      for (int i = 0; i < (blockDim.x >> 5); ++i) tot += s[i];
      norm_out[0] = sumsq_only ? tot : sqrtf(tot);
      if (user_norm && !sumsq_only) user_norm[0] = norm_out[0];
      *ticket = 0;
      counters[0] += 1;  // optax adam `count` (also counts rmsprop steps)
    }
  }
}

struct OptArgs {
  int kind; float lr, eps, decay, b1, b2, max_norm;
  float* p; const float* g; float* m; float* v; long long n; const float* norm; const int64_t* counters;
  // split global norm (tensor-core path): norm = sqrt(fc_sumsq[0] + sum of parts[0..nparts)), recomputed identically by every block
  const float* parts; int nparts; const float* fc_sumsq; float* norm_out; float* user_norm;
  int stages;   // optimizer_bulk_kernel: depth of the shared-memory ring
};

// Fixed-order block reduction of the split-norm partials: every block of every launch gets the same bits.
__device__ __forceinline__ float split_norm(const float* __restrict__ parts, int nparts, const float* __restrict__ fc_sumsq) {
  __shared__ float s_red[8];
  float t = 0.f;
  if (threadIdx.x < 256) {   // the first 256 threads reduce (blocks of 256 or 512 threads): one fixed order
    for (int i = threadIdx.x; i < nparts; i += 256) t += __ldcg(parts + i);
    t = warp_sum(t);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = t;
  }
  __syncthreads();
  float tot = __ldcg(fc_sumsq);
#pragma unroll
  for (int i = 0; i < 8; ++i) tot += s_red[i];
  return sqrtf(tot);
}

__global__ void __launch_bounds__(256) norm_finalize_kernel(const float* parts, int nparts, const float* fc_sumsq, float* norm_out,
                                                            float* user_norm) {
  dz::pdl_enter();
  const float norm = split_norm(parts, nparts, fc_sumsq);
  if (threadIdx.x == 0) { norm_out[0] = norm; if (user_norm) user_norm[0] = norm; }
}

// One parameter.  optax.scale_by_adam divides the moments by (1 - b^t) per element; here the two
// reciprocals are formed once per thread and multiplied in (<= 1 ulp from the division), leaving one sqrt
// and one division per parameter instead of four IEEE-division sequences: the kernel was issue-bound.
template <int KIND>
__device__ __forceinline__ float opt_one(const OptArgs& o, float p, float g, float& m, float& v, bool clip, float norm,
                                         float inv_c1, float inv_c2) {
  if (clip) g = (g / norm) * o.max_norm;
  float upd;
  if (KIND == DZ_ADAM) {  // optax.scale_by_adam: eps outside the sqrt, bias-corrected moments
    float mu = o.b1 * m + (1.0f - o.b1) * g;
    float nu = o.b2 * v + (1.0f - o.b2) * g * g;
    // Moments of parameters whose gradient stays zero decay THROUGH the denormal range (0.9^t reaches 1e-38 after ~800
    // steps) and every warp that holds one takes the slow paths of the IEEE division / square root below: measured, the
    // optimizer launch went 42.7 -> 58.5 us between step 50 and step 4000 of a run.  A denormal moment cannot change a
    // parameter (|update| < 1e-38 / eps), so it is stored as zero.
    if (fabsf(mu) < 1.17549435e-38f) mu = 0.f;
    if (nu < 1.17549435e-38f) nu = 0.f;
    m = mu; v = nu;
    upd = (mu * inv_c1) / (sqrtf(nu * inv_c2) + o.eps);
  } else {                // optax.rmsprop(centered=True): eps inside the sqrt
    float mu = o.decay * m + (1.0f - o.decay) * g;
    float nu = o.decay * v + (1.0f - o.decay) * g * g;
    if (fabsf(mu) < 1.17549435e-38f) mu = 0.f;   // see the Adam branch: no denormal moments in memory
    if (nu < 1.17549435e-38f) nu = 0.f;
    m = mu; v = nu;
    upd = g * (1.0f / sqrtf(nu - mu * mu + o.eps));
  }
  return p - o.lr * upd;
}

// The optimizer update (7 floats of traffic per parameter: read p, g, m, v; write p, m, v) as a bulk-copy (TMA 1-D)
// pipeline: the four streams of a 256-quadruple chunk land in shared memory by cp.async.bulk (one elected thread,
// mbarrier complete_tx), the threads update them in place, and p / m / v leave by cp.async.bulk stores.  Memory-level
// parallelism does not depend on registers x resident warps: every CTA keeps `stages` - 1 chunks (16 KB each) of loads
// in flight while it computes, and the LSU sees shared-memory traffic only.
constexpr int kOptChunk = 256;                            // float4 per stream per stage
constexpr int kOptStageBytes = 4 * kOptChunk * 16;        // p, g, m, v
constexpr int kOptRingStages = 3;                         // OptArgs::stages of every launch
constexpr int kOptSmem = kOptRingStages * kOptStageBytes + 64;   // the ring + its mbarriers
constexpr int kOptThreads = kOptChunk * 2;                // 2 floats per thread and stream
constexpr int kOptBlocksPerSM = 4;

template <int KIND>
__global__ void __launch_bounds__(kOptThreads, kOptBlocksPerSM) optimizer_bulk_kernel(OptArgs o) {
  extern __shared__ __align__(128) unsigned char opt_sm[];
  const int kOptStages = o.stages;
  uint64_t* full = reinterpret_cast<uint64_t*>(opt_sm + kOptStages * kOptStageBytes);
  const int tid = threadIdx.x;
  const long long n4 = o.n >> 2;
  const long long nchunks = (n4 + kOptChunk - 1) / kOptChunk;
  const long long mine = blockIdx.x < nchunks ? (nchunks - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;   // chunks of this CTA
  float4* p4 = reinterpret_cast<float4*>(o.p);
  const float4* g4 = reinterpret_cast<const float4*>(o.g);
  float4* m4 = reinterpret_cast<float4*>(o.m);
  float4* v4 = reinterpret_cast<float4*>(o.v);
  if (tid == 0) {
    for (int s = 0; s < kOptStages; ++s) mbar_init(&full[s], 1);
    fence_mbarrier_init();
  }
  __syncthreads();
  dz::pdl_enter();
  auto issue = [&](long long it, int s) {   // thread 0: loads of this CTA's it-th chunk into stage s = it % stages
    const long long c = blockIdx.x + it * gridDim.x;
    const long long q0 = c * kOptChunk;
    const uint32_t bytes = (uint32_t)(min((long long)kOptChunk, n4 - q0) * 16);
    const uint32_t st = smem_u32(opt_sm + s * kOptStageBytes);
    mbar_expect_tx(&full[s], 4 * bytes);
    bulk_g2s(st, p4 + q0, bytes, &full[s]);
    bulk_g2s(st + kOptChunk * 16, g4 + q0, bytes, &full[s]);
    bulk_g2s(st + 2 * kOptChunk * 16, m4 + q0, bytes, &full[s]);
    bulk_g2s(st + 3 * kOptChunk * 16, v4 + q0, bytes, &full[s]);
  };
  // the first loads are issued BEFORE the norm is formed: the split-norm reduction (shared memory, a block barrier,
  // ~700 L2 reads per block) then hides behind the memory latency of the stream instead of preceding it
  if (tid == 0)
    for (long long it = 0; it < mine && it < kOptStages; ++it) issue(it, (int)it);
  float norm;
  if (o.parts != nullptr) {
    norm = split_norm(o.parts, o.nparts, o.fc_sumsq);
    if (blockIdx.x == 0 && tid == 0) { o.norm_out[0] = norm; if (o.user_norm) o.user_norm[0] = norm; }
  } else {
    norm = o.norm[0];
  }
  const bool clip = o.max_norm > 0.f && !(norm < o.max_norm);  // optax.clip_by_global_norm trigger
  float c1 = 1.f, c2 = 1.f;
  if (KIND == DZ_ADAM) {
    float t = (float)o.counters[0];
    c1 = 1.0f / (1.0f - powf(o.b1, t));
    c2 = 1.0f / (1.0f - powf(o.b2, t));
  }
  int s = 0;
  uint32_t phase = 0;
  for (long long it = 0; it < mine; ++it) {
    const long long q0 = (blockIdx.x + it * gridDim.x) * (long long)kOptChunk;
    const int valid = (int)min((long long)kOptChunk, n4 - q0);
    float4* sp = reinterpret_cast<float4*>(opt_sm + s * kOptStageBytes);
    float4* sg = sp + kOptChunk;
    float4* smm = sp + 2 * kOptChunk;
    float4* sv = sp + 3 * kOptChunk;
    if (tid == 0 && it > 0) {   // refill the stage of iteration it - 1 as soon as its stores have finished READING it
      const long long next = it - 1 + kOptStages;
      if (next < mine) {
        bulk_wait_group_read();
        issue(next, s == 0 ? kOptStages - 1 : s - 1);
      }
    }
    mbar_wait(&full[s], phase);
    if (tid < 2 * valid) {
      float2 p = reinterpret_cast<float2*>(sp)[tid], g = reinterpret_cast<float2*>(sg)[tid];
      float2 m = reinterpret_cast<float2*>(smm)[tid], v = reinterpret_cast<float2*>(sv)[tid];
      p.x = opt_one<KIND>(o, p.x, g.x, m.x, v.x, clip, norm, c1, c2);
      p.y = opt_one<KIND>(o, p.y, g.y, m.y, v.y, clip, norm, c1, c2);
      reinterpret_cast<float2*>(sp)[tid] = p; reinterpret_cast<float2*>(smm)[tid] = m; reinterpret_cast<float2*>(sv)[tid] = v;
    }
    fence_proxy_async_shared();   // generic-proxy writes -> visible to the bulk stores
    __syncthreads();
    if (tid == 0) {
      const uint32_t bytes = (uint32_t)valid * 16;
      bulk_s2g(p4 + q0, sp, bytes);
      bulk_s2g(m4 + q0, smm, bytes);
      bulk_s2g(v4 + q0, sv, bytes);
      bulk_commit_group();
    }
    if (++s == kOptStages) { s = 0; phase ^= 1u; }
  }
  if (tid == 0) bulk_wait_group();   // stores complete before the grid does
}

using OptKernel = void (*)(OptArgs);
OptKernel optimizer_kernel_for(int kind) {
  return kind == DZ_ADAM ? optimizer_bulk_kernel<DZ_ADAM> : optimizer_bulk_kernel<DZ_RMSPROP_CENTERED>;
}

// The dueling head of up to three passes (blockIdx.y): one warp per row forms the advantages adv = h1_adv adv2/w +
// adv2/b and the value v = h1_val val2/w + val2/b, and writes q = dueling_aggregate(adv, v) to out.  Lane l owns the
// inputs k = l + 32 j (j = 0..15) and sums its 16 terms of each output in j order; an xor butterfly then adds the 32
// lanes' partials in a fixed order, which leaves every lane with the same bits.  No sum depends on how many rows the
// launch holds.  The advantages go four at a time, so that the 64 weight loads of four outputs are in flight together
// (the 8 warps of a block apply the same pass, so its weights are read from L1 after the first row).
struct DuelingFwdArgs {
  const float* h1[3][2];    // [rows][512] of each pass's advantage / value stream
  const float* params[3];   // each pass's parameter blob
  float* out[3];            // q [rows][A]
  long long off_w[2], off_b[2];
  int rows, A;
};

// The noisy dueling head (DESIGN.md §17): the same launch with each weight formed in registers as
// w = fmaf(sigma_w, eps_in_k * eps_out_a, mu_w) (the operations of gemm_nn_kernel<DUAL>) and each bias as
// b = fmaf(sigma_b, eps_out_a, mu_b), where mu_b is added before the sigma term as in its epilogue.
struct NoisyDuelingFwdArgs {
  DuelingFwdArgs h;
  long long off_sw[2], off_sb[2];
  const float* noise[3];    // each pass's noise apply
  long long noise_ld;       // floats between the applies of consecutive rows (per-stream acting); 0: one apply per pass
  long long off_in[2], off_out[2];   // offsets in an apply of each stream's head eps_in [512] / eps_out
};

__device__ __forceinline__ float warp_sum_xor(float s) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  return s;
}

template <bool NOISY>
__device__ __forceinline__ void dueling_head_fwd(const DuelingFwdArgs& h, const NoisyDuelingFwdArgs* n) {
  __shared__ float adv_s[8][kDuelingMaxActions];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, p = blockIdx.y, A = h.A;
  const long long r = (long long)blockIdx.x * 8 + warp;
  if (r >= h.rows) return;
  const float* __restrict__ xa = h.h1[p][0] + r * 512;
  const float* __restrict__ xv = h.h1[p][1] + r * 512;
  const float* __restrict__ P = h.params[p];
  const float* __restrict__ Wa = P + h.off_w[0];
  const float* __restrict__ Wv = P + h.off_w[1];
  const float *Sa = nullptr, *Sv = nullptr, *eia = nullptr, *eoa = nullptr, *eiv = nullptr;
  float eov = 0.f;
  if constexpr (NOISY) {
    const float* nz = n->noise[p] + r * n->noise_ld;
    Sa = P + n->off_sw[0]; Sv = P + n->off_sw[1];
    eia = nz + n->off_in[0]; eoa = nz + n->off_out[0]; eiv = nz + n->off_in[1]; eov = nz[n->off_out[1]];
  }
  float x[16];
  float ei[NOISY ? 16 : 1];
  float sv = 0.f;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    x[j] = xa[lane + 32 * j];
    if constexpr (NOISY) {
      const int k = lane + 32 * j;
      ei[j] = eia[k];
      sv = fmaf(xv[k], fmaf(Sv[k], eiv[k] * eov, Wv[k]), sv);
    } else {
      sv = fmaf(xv[lane + 32 * j], Wv[lane + 32 * j], sv);
    }
  }
  float v = warp_sum_xor(sv) + P[h.off_b[1]];
  if constexpr (NOISY) v = fmaf(P[n->off_sb[1]], eov, v);
  for (int a0 = 0; a0 < A; a0 += 4) {
    const int na = A - a0 < 4 ? A - a0 : 4;
    float s[4] = {0.f, 0.f, 0.f, 0.f};
    float eo[NOISY ? 4 : 1];
    if constexpr (NOISY) {
#pragma unroll
      for (int c = 0; c < 4; ++c) eo[c] = c < na ? eoa[a0 + c] : 0.f;
    }
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float* __restrict__ w = Wa + (long long)(lane + 32 * j) * A + a0;
      if constexpr (NOISY) {
        const float* __restrict__ sg = Sa + (long long)(lane + 32 * j) * A + a0;
#pragma unroll
        for (int c = 0; c < 4; ++c)
          if (c < na) s[c] = fmaf(x[j], fmaf(sg[c], ei[j] * eo[c], w[c]), s[c]);
      } else {
#pragma unroll
        for (int c = 0; c < 4; ++c)
          if (c < na) s[c] = fmaf(x[j], w[c], s[c]);
      }
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const float t = warp_sum_xor(s[c]);
      if constexpr (NOISY) {
        if (lane == 0 && c < na) adv_s[warp][a0 + c] = fmaf(P[n->off_sb[0] + a0 + c], eo[c], t + P[h.off_b[0] + a0 + c]);
      } else {
        if (lane == 0 && c < na) adv_s[warp][a0 + c] = t + P[h.off_b[0] + a0 + c];
      }
    }
  }
  __syncwarp();
  if (lane == 0) dueling_aggregate(adv_s[warp], v, A, adv_s[warp]);
  __syncwarp();
  for (int a = lane; a < A; a += 32) h.out[p][r * A + a] = adv_s[warp][a];
}

__global__ void __launch_bounds__(256) dueling_head_fwd_kernel(const __grid_constant__ DuelingFwdArgs h) {
  dz::pdl_enter();
  dueling_head_fwd<false>(h, nullptr);
}

__global__ void __launch_bounds__(256) noisy_dueling_head_fwd_kernel(const __grid_constant__ NoisyDuelingFwdArgs n) {
  dz::pdl_enter();
  dueling_head_fwd<true>(n.h, &n);
}

// The dueling head's backward of online(s_tm1), one warp per row: dadv and dval from dq (dueling_transpose; dadv
// overwrites dq in place and dval goes to its own [B] buffer, both for the head weight gradients), then both streams'
// dh1: dh1_adv = dadv adv2/w^T and dh1_val = dval val2/w^T, each masked by its own h1 > 0.  Lane l owns inputs
// k = l + 32 j; dh1_adv[k] sums serially over the actions, the 16 inputs of a lane side by side so that their weight
// loads are in flight together.  With hi / lo set it also writes the tf32 hi/lo pair of both streams that the
// tensor-core input gradient reads.
struct DuelingBwdArgs {
  float* dq;                 // [B][A]: in dq, out dadv
  float* dval;               // [B]
  const float* h1[2];        // [B][512] post-ReLU activations of online(s_tm1), the masks
  const float* W[2];         // adv2/w [512][A], val2/w [512][1] of the online blob
  float* dh1[2];             // [B][512]
  float *hi[2], *lo[2];      // optional tf32 images of dh1, same layout
  int B, A;
};

// The noisy dueling head's backward: the same launch through the weights the forward formed (noise apply 0).
struct NoisyDuelingBwdArgs {
  DuelingBwdArgs g;
  const float* S[2];                    // adv2/sigma/w, val2/sigma/w of the online blob
  const float *ein[2], *eout[2];        // each stream's head eps_in [512] / eps_out
};

template <bool NOISY>
__device__ __forceinline__ void dueling_head_bwd(const DuelingBwdArgs& g, const NoisyDuelingBwdArgs* n) {
  __shared__ float d_s[8][kDuelingMaxActions + 1];   // per warp: [0, A) dadv, [kDuelingMaxActions] dval
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, A = g.A;
  const long long r = (long long)blockIdx.x * 8 + warp;
  if (r >= g.B) return;
  float* __restrict__ d = d_s[warp];
  for (int a = lane; a < A; a += 32) d[a] = g.dq[r * A + a];
  __syncwarp();
  if (lane == 0) d[kDuelingMaxActions] = dueling_transpose(d, A, d);
  __syncwarp();
  for (int a = lane; a < A; a += 32) g.dq[r * A + a] = d[a];
  const float dval = d[kDuelingMaxActions];
  if (lane == 0) g.dval[r] = dval;
  const float* __restrict__ Wa = g.W[0];
  const float* __restrict__ Wv = g.W[1];
  float acc[16];
  float ei[NOISY ? 16 : 1];
#pragma unroll
  for (int j = 0; j < 16; ++j) acc[j] = 0.f;
  if constexpr (NOISY) {
#pragma unroll
    for (int j = 0; j < 16; ++j) ei[j] = n->ein[0][lane + 32 * j];
  }
#pragma unroll 2
  for (int a = 0; a < A; ++a) {
    const float da = d[a];
    if constexpr (NOISY) {
      const float eo = n->eout[0][a];
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const long long i = (long long)(lane + 32 * j) * A + a;
        acc[j] = fmaf(da, fmaf(n->S[0][i], ei[j] * eo, Wa[i]), acc[j]);
      }
    } else {
#pragma unroll
      for (int j = 0; j < 16; ++j) acc[j] = fmaf(da, Wa[(long long)(lane + 32 * j) * A + a], acc[j]);
    }
  }
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int k = lane + 32 * j;
    const long long i = r * 512 + k;
    const float va = g.h1[0][i] > 0.f ? acc[j] : 0.f;
    float vv;
    if constexpr (NOISY) vv = g.h1[1][i] > 0.f ? dval * fmaf(n->S[1][k], n->ein[1][k] * n->eout[1][0], Wv[k]) : 0.f;
    else vv = g.h1[1][i] > 0.f ? dval * Wv[k] : 0.f;
    g.dh1[0][i] = va;
    g.dh1[1][i] = vv;
    if (g.hi[0]) {
      float hi, lo;
      tc::split_tf32(va, hi, lo);
      g.hi[0][i] = hi; g.lo[0][i] = lo;
      tc::split_tf32(vv, hi, lo);
      g.hi[1][i] = hi; g.lo[1][i] = lo;
    }
  }
}

__global__ void __launch_bounds__(256) dueling_head_bwd_kernel(const __grid_constant__ DuelingBwdArgs g) {
  dz::pdl_enter();
  dueling_head_bwd<false>(g, nullptr);
}

__global__ void __launch_bounds__(256) noisy_dueling_head_bwd_kernel(const __grid_constant__ NoisyDuelingBwdArgs n) {
  dz::pdl_enter();
  dueling_head_bwd<true>(n.g, &n);
}

// ---- Rainbow's noisy head (DESIGN.md §7): two streams (advantage 512 -> A * atoms, value 512 -> atoms) without a split
// reduction or a finish launch.  Each weight is formed as fmaf(sigma_w, eps_in_k * eps_out_n, mu_w), the operations of
// gemm_nn_kernel<DUAL> / gemm_nt_kernel<DUAL>.

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem)), "l"(gmem));
}
__device__ __forceinline__ void cp_async4(void* smem, const void* gmem) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((uint32_t)__cvta_generic_to_shared(smem)), "l"(gmem));
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

constexpr int kNhTile = 8;       // forward: output columns of one stream per CTA
constexpr int kNhRows = 32;      // forward: rows (images) per pass
constexpr int kNhLd = 68;        // forward: x row stride in shared memory, 17 16-byte units (odd: conflict-free float4 reads)
constexpr int kNhKc = 4;         // backward: dh1 columns per CTA
constexpr size_t kMaxDynSmem = 227 * 1024;   // the most dynamic shared memory one CTA may opt in to
constexpr size_t kNhFwdSmem = (size_t)(8 * 2 * kNhRows * kNhLd + 8 * 2 * 64 * kNhTile) * sizeof(float);

// Forward.  blockIdx.y is a group of one or two passes that apply the same parameter blob (online on s_tm1 and s_t,
// target on s_t): the group's CTAs read each mu / sigma tile once and form it with every member's noise.  blockIdx.x
// is a kNhTile-column tile of stream 0's outputs, then of stream 1's.  Warp w reduces k in [64 w, 64 w + 64) for all
// rows, columns and members in ascending k order; the eight warp sums are then added in warp order, then mu_b (if any)
// and fmaf(sigma_b, eps_out, .) as finish_nn_body does.  The order depends on nothing but k.
struct NoisyHeadFwdArgs {
  const float* x[2][2][2];        // [group][member][stream]: h1 [rows][512]
  float* out[2][2][2];            // [group][member][stream]: [rows][N[stream]]
  const float* ein[2][2][2];      // [group][member][stream]: eps_in [512]
  const float* eout[2][2][2];     // [group][member][stream]: eps_out [N[stream]]
  const float* mu[2][2];          // [group][stream]: [512][N]
  const float* sigma[2][2];
  const float* bias[2][2];        // mu bias [N] (or [1] with bias_shared), nullptr without one
  const float* sbias[2][2];       // sigma bias [N]
  int members[2];
  int N[2], tiles0;               // stream widths; tiles of stream 0
  int rows, bias_shared;
};

template <int P>
__device__ __forceinline__ void noisy_head_fwd(const NoisyHeadFwdArgs& a) {
  extern __shared__ __align__(16) float nh_smem[];
  const int g = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int s = (int)blockIdx.x < a.tiles0 ? 0 : 1;
  const int n0 = (s == 0 ? (int)blockIdx.x : (int)blockIdx.x - a.tiles0) * kNhTile, N = a.N[s];
  const int k0 = warp * 64;
  float* xs = nh_smem + warp * (2 * kNhRows * kNhLd);                      // [P][rows][kNhLd]: this warp's k slice
  float* ws = nh_smem + 8 * 2 * kNhRows * kNhLd + warp * (2 * 64 * kNhTile);  // [P][64][kNhTile]: formed weights
  // this thread's bias terms in the final sums (column n0 + threadIdx.x % kNhTile, member q), loaded up front
  const int ne = n0 + (int)(threadIdx.x % kNhTile);
  float bias_e = 0.f, sb_e = 0.f, eo_e[P];
  if (ne < N) {
    const float* b = a.bias[g][s];
    if (b) bias_e = a.bias_shared ? b[0] : b[ne];
    sb_e = a.sbias[g][s][ne];
  }
#pragma unroll
  for (int q = 0; q < P; ++q) eo_e[q] = ne < N ? a.eout[g][q][s][ne] : 0.f;
  for (int p = 0; p < P; ++p) {
    const float* x = a.x[g][p][s];
    for (int i = lane; i < kNhRows * 16; i += 32) {
      const int m = i >> 4, q = (i & 15) * 4;
      float* dst = xs + (p * kNhRows + m) * kNhLd + q;
      if (m < a.rows) cp_async16(dst, x + (long long)m * 512 + k0 + q);
      else *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  {
    // every load of the tile is issued before any is used: the weights come from HBM, and a loop that waited for
    // them a few rows at a time paid their latency once per few rows
    const int c = lane & 7, n = n0 + c, kr = lane >> 3;
    const bool ok = n < N;
    const float* __restrict__ mu = a.mu[g][s];
    const float* __restrict__ sg = a.sigma[g][s];
    float m_[16], s_[16], ei[P][16], eo[P];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int k = k0 + kr + 4 * i;
      m_[i] = ok ? mu[(long long)k * N + n] : 0.f;
      s_[i] = ok ? sg[(long long)k * N + n] : 0.f;
#pragma unroll
      for (int p = 0; p < P; ++p) ei[p][i] = a.ein[g][p][s][k];
    }
#pragma unroll
    for (int p = 0; p < P; ++p) eo[p] = ok ? a.eout[g][p][s][n] : 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i)
#pragma unroll
      for (int p = 0; p < P; ++p) ws[(p * 64 + kr + 4 * i) * kNhTile + c] = fmaf(s_[i], ei[p][i] * eo[p], m_[i]);
  }
  cp_async_wait_all();
  __syncwarp();
  // lane: row group rg (rows rg + RG i), column quad cq, member p
  constexpr int RM = 2 * P, RG = kNhRows / RM;
  const int rg = lane % RG, cq = (lane / RG) & 1, p = lane / (2 * RG);
  float acc[RM][4];
#pragma unroll
  for (int i = 0; i < RM; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  const float* xp = xs + (p * kNhRows + rg) * kNhLd;
  const float* wp = ws + p * 64 * kNhTile + cq * 4;
#pragma unroll 4
  for (int kq = 0; kq < 64; kq += 4) {
    float4 xv[RM];
#pragma unroll
    for (int i = 0; i < RM; ++i) xv[i] = *reinterpret_cast<const float4*>(xp + i * RG * kNhLd + kq);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float4 w = *reinterpret_cast<const float4*>(wp + (kq + e) * kNhTile);
#pragma unroll
      for (int i = 0; i < RM; ++i) {
        const float xe = e == 0 ? xv[i].x : e == 1 ? xv[i].y : e == 2 ? xv[i].z : xv[i].w;
        acc[i][0] = fmaf(xe, w.x, acc[i][0]); acc[i][1] = fmaf(xe, w.y, acc[i][1]);
        acc[i][2] = fmaf(xe, w.z, acc[i][2]); acc[i][3] = fmaf(xe, w.w, acc[i][3]);
      }
    }
  }
  __syncwarp();
  float* red = xs;   // [P][rows][kNhTile] warp sums, over this warp's own x slice
#pragma unroll
  for (int i = 0; i < RM; ++i)
    *reinterpret_cast<float4*>(red + (p * kNhRows + rg + i * RG) * kNhTile + cq * 4) =
        make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
  __syncthreads();
#pragma unroll
  for (int q = 0; q < P; ++q) {   // 256 threads: t = q * 256 + threadIdx.x covers [P][rows][kNhTile]
    const int t = q * kNhRows * kNhTile + (int)threadIdx.x, m = (int)threadIdx.x / kNhTile;
    if (m >= a.rows || ne >= N) continue;
    float v = nh_smem[t];
#pragma unroll
    for (int w = 1; w < 8; ++w) v += nh_smem[w * (2 * kNhRows * kNhLd) + t];
    if (a.bias[g][s]) v += bias_e;
    v = fmaf(sb_e, eo_e[q], v);
    a.out[g][q][s][(long long)m * N + ne] = v;
  }
}

// Both head kernels let the next kernel launch as soon as every CTA is resident: its launch and set-up overlap this
// kernel, and its griddepcontrol.wait (every kernel's first step) still waits for this grid to complete.
__device__ __forceinline__ void noisy_head_enter() {
  dz::pdl_enter();
  if (threadIdx.x == 0) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

__global__ void __launch_bounds__(256) noisy_head_fwd_kernel(const __grid_constant__ NoisyHeadFwdArgs a) {
  noisy_head_enter();
  if (a.members[blockIdx.y] == 2) noisy_head_fwd<2>(a);
  else noisy_head_fwd<1>(a);
}

// Input gradient through online(s_tm1)'s head (noise apply 0): dh1_s[m][k] = sum_n dout_s[m][n] W_s[k][n], masked by
// h1_s > 0, for both streams; CTA j owns k in [kNhKc j, kNhKc j + kNhKc).  The CTA stages every row of dout and forms
// its weights in shared memory; each warp then takes four rows at a time: lane l sums n = l + 32 i in ascending i for
// the 32 outputs (4 rows x 2 streams x kNhKc columns), and a halving butterfly leaves output l's total in lane l.  The
// order depends on nothing but n.  With hi / lo set it also writes the tf32 hi/lo pair the tensor-core fc1 input
// gradient reads, as finish_nt_kernel does.
struct NoisyHeadBwdArgs {
  const float* dout[2];           // [B][N[s]]
  const float* mu[2];             // [512][N[s]] of the online blob
  const float* sigma[2];
  const float* ein[2];            // eps_in [512]
  const float* eout[2];           // eps_out [N[s]]
  const float* h1[2];             // [B][512], the masks
  float* dh1[2];                  // [B][512]
  float *hi[2], *lo[2];           // optional tf32 images of dh1
  int N[2], B;
};

// acc[r * 8 + S * kNhKc + kl] += sum over lane's n of d[m0 + r][n] w[kl][n] (stream S: d [B][N], w row stride NT).
template <int S>
__device__ __forceinline__ void noisy_head_bwd_sum(float (&acc)[32], const float* d, const float* w, int N, int NT, int B,
                                                   int m0, int lane) {
  for (int n = lane; n < N; n += 32) {
    float wk[kNhKc];
#pragma unroll
    for (int kl = 0; kl < kNhKc; ++kl) wk[kl] = w[kl * NT + n];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const float dv = m0 + r < B ? d[(m0 + r) * N + n] : 0.f;
#pragma unroll
      for (int kl = 0; kl < kNhKc; ++kl) acc[r * 8 + S * kNhKc + kl] = fmaf(dv, wk[kl], acc[r * 8 + S * kNhKc + kl]);
    }
  }
}

// One step of the halving butterfly: lanes with bit H set keep outputs [H, 2H) of acc, the others [0, H); each adds its
// partner's partial sums of the half it keeps.
template <int H>
__device__ __forceinline__ void noisy_head_halve(float (&acc)[32], int lane) {
  const bool up = (lane & H) != 0;
#pragma unroll
  for (int o = 0; o < H; ++o) {
    const float a0 = acc[o], a1 = acc[o + H];
    acc[o] = (up ? a1 : a0) + __shfl_xor_sync(0xffffffffu, up ? a0 : a1, H);
  }
}

__global__ void __launch_bounds__(256) noisy_head_bwd_kernel(const __grid_constant__ NoisyHeadBwdArgs a) {
  noisy_head_enter();
  extern __shared__ __align__(16) float nh_smem[];
  const int N0 = a.N[0], N1 = a.N[1], NT = N0 + N1, B = a.B;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, k0 = blockIdx.x * kNhKc;
  float* ds = nh_smem;                  // [B][N0] then [B][N1]
  float* ws = nh_smem + (long long)B * NT;   // [kNhKc][N0 + N1]: stream 0's columns, then stream 1's
  for (int i = threadIdx.x; i < B * N0; i += blockDim.x) cp_async4(ds + i, a.dout[0] + i);
  for (int i = threadIdx.x; i < B * N1; i += blockDim.x) cp_async4(ds + B * N0 + i, a.dout[1] + i);
  // the weights come from HBM: eight of each thread's elements are loaded before any is used, so that their latency
  // is paid once per 8 x 256 elements (rainbow: 4 x 357, once)
  for (int i0 = threadIdx.x; i0 < kNhKc * NT; i0 += 8 * 256) {
    float m_[8], s_[8], e_[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int i = i0 + j * 256;
      m_[j] = s_[j] = e_[j] = 0.f;
      if (i < kNhKc * NT) {
        const int kl = i / NT, c = i % NT, s = c < N0 ? 0 : 1, n = s ? c - N0 : c, k = k0 + kl;
        const long long wi = (long long)k * a.N[s] + n;
        m_[j] = a.mu[s][wi]; s_[j] = a.sigma[s][wi]; e_[j] = a.ein[s][k] * a.eout[s][n];
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (i0 + j * 256 < kNhKc * NT) ws[i0 + j * 256] = fmaf(s_[j], e_[j], m_[j]);
  }
  cp_async_wait_all();
  __syncthreads();
  for (int m0 = warp * 4; m0 < B; m0 += 32) {
    float acc[32];   // acc[r * 8 + s * kNhKc + kl]
#pragma unroll
    for (int o = 0; o < 32; ++o) acc[o] = 0.f;
    noisy_head_bwd_sum<0>(acc, ds, ws, N0, NT, B, m0, lane);
    noisy_head_bwd_sum<1>(acc, ds + B * N0, ws + N0, N1, NT, B, m0, lane);
    // halving butterfly: after the step of width H, lane l holds in acc[0 .. H) the partial sums of the outputs whose
    // bit H matches l's
    noisy_head_halve<16>(acc, lane); noisy_head_halve<8>(acc, lane); noisy_head_halve<4>(acc, lane);
    noisy_head_halve<2>(acc, lane); noisy_head_halve<1>(acc, lane);
    const int r = lane >> 3, s = (lane >> 2) & 1, kl = lane & 3, m = m0 + r, k = k0 + kl;
    if (m < B) {
      const long long i = (long long)m * 512 + k;
      const float v = a.h1[s][i] > 0.f ? acc[0] : 0.f;
      a.dh1[s][i] = v;
      if (a.hi[s]) {
        float hi, lo;
        tc::split_tf32(v, hi, lo);
        a.hi[s][i] = hi; a.lo[s][i] = lo;
      }
    }
  }
}

// epsilon-greedy over q[E][A] (dqn/agent.py:121-127): first maximum wins, as np.argmax / jnp.argmax.
__global__ void act_select_kernel(const float* __restrict__ q, int A, int E, const float* __restrict__ explore, float eps,
                                  int32_t* __restrict__ actions) {
  dz::pdl_enter();
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  int best = 0;
  float bq = q[(long long)e * A];
  for (int a = 1; a < A; ++a) {
    const float v = q[(long long)e * A + a];
    if (v > bq) { bq = v; best = a; }
  }
  if (explore != nullptr && explore[e] < eps) best = min((int)(explore[E + e] * (float)A), A - 1);
  actions[e] = best;
}

__global__ void make_row_table_kernel(const uint8_t* base, long long stride, int n, const uint8_t** table) {
  dz::pdl_enter();
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) table[i] = base + (long long)i * stride;
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// The learner object
// ------------------------------------------------------------------------------------------------

// A stream beside the caller's, joined back by events; under stream capture it becomes a parallel branch of the CUDA graph.
struct SideStream {
  cudaStream_t stream = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  bool dirty = false;   // work was enqueued since the last join

  cudaError_t create() {
    cudaError_t e = cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ev_join, cudaEventDisableTiming);
    return e;
  }
  void destroy() {
    if (stream) { cudaStreamSynchronize(stream); cudaStreamDestroy(stream); }
    if (ev_fork) cudaEventDestroy(ev_fork);
    if (ev_join) cudaEventDestroy(ev_join);
  }
  // Returns the side stream after making it wait for everything enqueued on `from` so far, or `fallback` when that
  // ordering cannot be recorded.
  void* fork(void* from, void* fallback) {
    if (cudaEventRecord(ev_fork, (cudaStream_t)from) != cudaSuccess) return fallback;
    if (cudaStreamWaitEvent(stream, ev_fork, 0) != cudaSuccess) return fallback;
    dirty = true;
    return stream;
  }
  // Makes `into` wait for the side work enqueued since the last join.
  int join(void* into) {
    if (!dirty) return DZ_OK;
    DZ_CUDA_OK(cudaEventRecord(ev_join, stream));
    DZ_CUDA_OK(cudaStreamWaitEvent((cudaStream_t)into, ev_join, 0));
    dirty = false;
    return DZ_OK;
  }
  // Where work that must follow the latest side work goes: the side stream while it has unjoined work, else `main`.
  void* tail(void* main) const { return dirty ? (void*)stream : main; }
};

struct dz_learner {
  dz_learner_config cfg;
  dz_learner_buffers buf;
  Layout lay;
  ParamOffsets po;
  Dims d;
  FcNet fc;        // the layers after the torso
  int B;           // train batch
  int n_head[3];   // rows per image in the head stage for pass 0/1/2 (IQN: tau samples; others 1)
  // workspace (floats unless noted)
  float *act1[3], *act2[3], *act3[3];
  float *h1[3][2], *out[3], *outv[3];      // rainbow: h1[p][0]=adv stream, [1]=val stream; out=adv, outv=val
  float *cosf[3], *hi[3], *E0;             // iqn
  // fqf: the step's proposals (application 0 = online(s_tm1)'s features, 1 = target(s_t)'s): fq_tau [2][B][N+1],
  // fq_hat / fq_w / fq_q [2][B][N]; the head passes' tau inputs fq_pass1 [B][N] and fq_pass2 [B][2N] (pass 0 reads
  // fq_hat[0]); the fraction logits' gradient fq_dlogits [B][N]; acting's tau_hat / w, fq_act_hat / fq_act_w [B][N]
  float *fq_tau, *fq_hat, *fq_w, *fq_q, *fq_pass1, *fq_pass2, *fq_dlogits, *fq_act_hat, *fq_act_w;
  float* nn_partial;                        // split-K partials for the M=batch FC layers and heads
  float* conv_partial;                      // split-K partials for conv2/conv3 forward
  float* nt_partial;                        // split partials of the input-gradient (NT) GEMMs
  float *dout, *doutv, *dh1[2], *dact3, *dcol, *dact2, *dact1, *dhi;
  float* tn_partial[4];                     // conv1/2/3 wgrad partials, [3] = iqn head/embed partial
  float *loss_terms, *scalars;              // scalars: [0]=norm, [1]=shared-bias scratch.., [8..]=norm partials
  unsigned int* ticket;
  const uint8_t** rows_sample[2];           // row tables filled by the fused sampler
  uint8_t* recon = nullptr;                 // frame-deduplicated replay: [B][2][obs_stride] stacks the sampled rows
  int64_t recon_bytes = 0;                  //   are rebuilt into (allocated by the first, eager, dz_learner_learn)
  // random_shift_pad > 0 (DESIGN.md §18): the step's shifted observations [B][2][obs_bytes] and the row tables of
  // s_tm1 / s_t into them, which the torso reads in place of the sampler's or the caller's
  uint8_t* shift_obs;
  const uint8_t** rows_shift[2];
  const uint8_t** rows_act;                 // [batch] observation row table of the learner's acting
  int32_t* s_a; float *s_r, *s_d, *s_w;     // sampler-produced batch scalars
  float* q_scratch;
  int fc_splits, head_splits, conv_splits, nt_splits;
  // packed-operand tensor-core path of the IQN 3136->512 layer (dz_tcp.cuh): hi/lo tile images + split partials
  bool pk_on;
  struct PkImg { float* hi; float* lo; int rows_pad, red_pad; };
  PkImg pk_act[3], pk_wT[2], pk_w, pk_actT, pk_dh1T, pk_dh1, pk_cos[3], pk_weT[2], pk_dET, pk_cosT;
  bool pk_embed_bwd;
  int pk_embed_wgrad_splits;
  float *pk_fwd_partial, *pk_wgrad_partial;
  int pk_fwd_splits, pk_wgrad_splits;
  // second stream for work that is off the critical path of the backward pass (weight gradients, priority
  // write-back, noise generation)
  SideStream side;
  // third branch: the conv2 weight gradient runs beside the first side stream
  SideStream side2;
  // fourth branch: the conv3 and conv1 weight gradients.  They need only the main stream's input gradients, so they
  // do not queue behind the FC / head weight gradients and the FC norm on the first side stream.
  SideStream side3;
  float* norm_parts;                        // split-norm slots written by the conv weight-gradient finish kernels
  // TMA-fed tensor-core path of the batch-sized step (dz_umma_net.cu): torso + 3136 -> 512 layer(s), forward and input gradients
  UmNet* um;
  char* um_ws;
  int um_npass;
  // The optimizer kernel's dynamic shared-memory limit is raised per learner (the attribute is per device) at the
  // learner's first optimizer launch, not at creation: raising it loads the kernel (CUDA lazy loading), and loading it
  // at creation left the dqn CUDA-graph step about 1% slower in most processes (measured on an H100 80GB HBM3 at 700 W,
  // with every kernel's code unchanged).
  bool opt_smem_set = false;
};

namespace {

constexpr int kNormBlocks = kNumSMs * 4;

// Split count for a one-CTA-per-SM kernel: minimise (waves of kNumSMs CTAs) x (k-blocks per split).
int pick_splits(int64_t tiles, int nkb, int max_splits) {
  int best = 1;
  int64_t best_cost = -1;
  for (int s = 1; s <= max_splits; ++s) {
    int64_t cost = ceil_div(tiles * s, kNumSMs) * (ceil_div(nkb, s) + 6);   // +6: pipeline fill/drain per CTA
    if (best_cost < 0 || cost < best_cost) { best_cost = cost; best = s; }
  }
  return best;
}

UmNetDesc make_um_desc(const dz_learner* l);

int64_t carve(dz_learner* l, char* base) {
  const dz_learner_config& c = l->cfg;
  const Dims& d = l->d;
  const int B = c.batch;
  Bump w{base};
  const FcNet& f = l->fc;
  const bool two = f.ns == 2, gemm_val = two && !f.dueling_head, iqn = uses_iqn_net(c.kind);
  int nh[3] = {1, 1, 1};
  if (draws_taus(c.kind)) { nh[0] = c.tau_samples_s_tm1; nh[1] = c.tau_samples_policy; nh[2] = c.tau_samples_s_t; }
  // fqf: online(s_tm1) at tau_hat | online(s_tm1) at tau_1..tau_N | target(s_t) at [tau_hat' | tau_hat]; acting uses pass 1
  if (proposes_fractions(c.kind)) { nh[0] = c.num_fractions; nh[1] = c.num_fractions; nh[2] = 2 * c.num_fractions; }
  for (int p = 0; p < 3; ++p) l->n_head[p] = nh[p];
  for (int p = 0; p < 3; ++p) {
    l->act1[p] = w.take<float>((int64_t)B * d.h1 * d.w1 * 32);
    l->act2[p] = w.take<float>((int64_t)B * d.h2 * d.w2 * 64);
    l->act3[p] = w.take<float>((int64_t)B * d.feat);
    int64_t rows = (int64_t)B * nh[p];
    l->h1[p][0] = w.take<float>(rows * 512);
    l->h1[p][1] = two ? w.take<float>(rows * 512) : nullptr;
    l->out[p] = w.take<float>(rows * d.out);
    l->outv[p] = gemm_val ? w.take<float>((int64_t)B * f.out[1]) : nullptr;
    l->cosf[p] = iqn ? w.take<float>(rows * c.latent_dim) : nullptr;
    l->hi[p] = iqn ? w.take<float>(rows * d.feat) : nullptr;
  }
  l->E0 = iqn ? w.take<float>((int64_t)B * nh[0] * d.feat) : nullptr;
  {
    const bool fq = proposes_fractions(c.kind);
    const int64_t n = fq ? (int64_t)B * c.num_fractions : 0;
    l->fq_tau = fq ? w.take<float>(2 * (n + B)) : nullptr;
    l->fq_hat = fq ? w.take<float>(2 * n) : nullptr;
    l->fq_w = fq ? w.take<float>(2 * n) : nullptr;
    l->fq_q = fq ? w.take<float>(2 * n) : nullptr;
    l->fq_pass1 = fq ? w.take<float>(n) : nullptr;
    l->fq_pass2 = fq ? w.take<float>(2 * n) : nullptr;
    l->fq_dlogits = fq ? w.take<float>(n) : nullptr;
    l->fq_act_hat = fq ? w.take<float>(n) : nullptr;
    l->fq_act_w = fq ? w.take<float>(n) : nullptr;
  }
  l->fc_splits = 14; l->head_splits = 8; l->conv_splits = 4; l->nt_splits = 8;
  {
    int64_t head_n = std::max<int64_t>(d.out, c.num_atoms);
    int64_t fc = (int64_t)kMaxProblems * l->fc_splits * 2 * B * 512;
    int64_t hd = (int64_t)kMaxProblems * l->head_splits * 2 * B * head_n;
    l->nn_partial = w.take<float>(std::max(fc, hd));
    l->conv_partial = w.take<float>((int64_t)3 * l->conv_splits * B * d.h2 * d.w2 * 64);
    l->nt_partial = w.take<float>((int64_t)2 * l->nt_splits * 2 * B * std::max<int64_t>(d.feat, 512));
  }
  int64_t rows0 = (int64_t)B * nh[0];
  l->dout = w.take<float>(rows0 * d.out);
  // the value stream's output gradient: rainbow's [B][atoms], the dueling network's dval [B]
  l->doutv = two ? w.take<float>((int64_t)B * f.out[1]) : nullptr;
  l->dh1[0] = w.take<float>(rows0 * 512);
  l->dh1[1] = two ? w.take<float>(rows0 * 512) : nullptr;
  l->dact3 = w.take<float>((int64_t)B * d.feat);
  int64_t col2 = (int64_t)B * d.h2 * d.w2 * 512, col3 = (int64_t)B * d.h3 * d.w3 * 576;
  l->dcol = w.take<float>(col2 > col3 ? col2 : col3);
  l->dact2 = w.take<float>((int64_t)B * d.h2 * d.w2 * 64);
  l->dact1 = w.take<float>((int64_t)B * d.h1 * d.w1 * 32);
  l->dhi = iqn ? w.take<float>(rows0 * d.feat) : nullptr;
  l->tn_partial[0] = w.take<float>((int64_t)64 * 257 * 32);
  l->tn_partial[1] = w.take<float>((int64_t)32 * 513 * 64);
  l->tn_partial[2] = w.take<float>((int64_t)32 * 577 * 64);
  l->tn_partial[3] = iqn ? w.take<float>((int64_t)16 * (c.latent_dim + 1) * d.feat + 16 * 513 * 64) : nullptr;
  l->pk_on = false; l->pk_embed_bwd = false;
  // The packed-operand tensor-core kernels carry IQN's 3136->512 layer whenever every network apply has >= 1024 rows.
  if (iqn && rows0 >= 1024 && (int64_t)B * nh[1] >= 1024 && (int64_t)B * nh[2] >= 1024 && d.feat % 16 == 0 &&
      c.latent_dim <= 128 && rows0 % 4 == 0 && ((int64_t)B * nh[1]) % 4 == 0 && ((int64_t)B * nh[2]) % 4 == 0) {
    l->pk_on = true;
    auto img = [&](dz_learner::PkImg& im, int64_t rows, int64_t red, int row_tile) {
      im.rows_pad = (int)(ceil_div(rows, row_tile) * row_tile);
      im.red_pad = (int)(ceil_div(red, kPkKB) * kPkKB);
      im.hi = w.take<float>(pk_image_floats(im.rows_pad, im.red_pad));
      im.lo = w.take<float>(pk_image_floats(im.rows_pad, im.red_pad));
    };
    int64_t tiles = 0;
    for (int p = 0; p < 3; ++p) { img(l->pk_act[p], (int64_t)B * nh[p], d.feat, 128); tiles += l->pk_act[p].rows_pad / 128 * 2; }
    img(l->pk_wT[0], 512, d.feat, 256);
    img(l->pk_wT[1], 512, d.feat, 256);
    img(l->pk_w, d.feat, 512, 256);
    img(l->pk_actT, d.feat + 1, rows0, 128);
    img(l->pk_dh1T, 512, rows0, 256);
    img(l->pk_dh1, rows0, 512, 128);
    for (int p = 0; p < 3; ++p) img(l->pk_cos[p], (int64_t)B * nh[p], c.latent_dim, 128);
    img(l->pk_weT[0], d.feat, c.latent_dim, 256);
    img(l->pk_weT[1], d.feat, c.latent_dim, 256);
    l->pk_embed_bwd = nh[0] == 64 && d.feat % 64 == 0;
    if (l->pk_embed_bwd) {
      img(l->pk_dET, d.feat, rows0, 128);
      img(l->pk_cosT, c.latent_dim + 1, rows0, 256);
      l->pk_embed_wgrad_splits = pick_splits(l->pk_dET.rows_pad / 128, l->pk_dET.red_pad / kPkKB, 8);
    }
    l->pk_fwd_splits = pick_splits(tiles, l->pk_act[0].red_pad / kPkKB, 6);
    l->pk_wgrad_splits = pick_splits((int64_t)l->pk_actT.rows_pad / 128 * 2, l->pk_actT.red_pad / kPkKB, 8);
    int64_t fwd_rows = (int64_t)B * (nh[0] + nh[1] + nh[2]);
    l->pk_fwd_partial = w.take<float>((int64_t)l->pk_fwd_splits * fwd_rows * 512);
    l->pk_wgrad_partial = w.take<float>((int64_t)l->pk_wgrad_splits * (d.feat + 1) * 512);
  }
  l->loss_terms = w.take<float>(B);
  l->scalars = w.take<float>(8 + kNormBlocks + d.out + 64);
  l->ticket = w.take<unsigned int>(4);
  l->rows_sample[0] = w.take<const uint8_t*>(B);
  l->rows_sample[1] = w.take<const uint8_t*>(B);
  l->rows_act = w.take<const uint8_t*>(B > 4 ? B : 4);
  l->s_a = w.take<int32_t>(B);
  l->s_r = w.take<float>(B);
  l->s_d = w.take<float>(B);
  l->s_w = w.take<float>(B);
  l->q_scratch = w.take<float>(64);
  l->norm_parts = w.take<float>(1024);
  l->um_ws = nullptr;
  UmNetDesc ud = make_um_desc(l);
  if (um_net_supported(ud)) {
    int64_t bytes = um_net_workspace_bytes(ud);
    l->um_ws = w.take<char>(bytes);
    if (!base) l->um_ws = reinterpret_cast<char*>(1);   // size query: "enabled" marker only
  }
  // last, so that with the pad at 0 the workspace and every offset in it are what they are without augmentation
  const bool shift = c.random_shift_pad > 0;
  l->shift_obs = shift ? w.take<uint8_t>((int64_t)B * 2 * d.H * d.W * d.C) : nullptr;   // H*W*C: a multiple of 16
  l->rows_shift[0] = shift ? w.take<const uint8_t*>(B) : nullptr;
  l->rows_shift[1] = shift ? w.take<const uint8_t*>(B) : nullptr;
  return w.used;
}

// A learner with cfg's configuration, layout, parameter offsets, network description, dims and split counts and no
// device state: carve() without a base leaves every workspace pointer NULL.  Returns the workspace bytes.
int64_t init_shape_learner(dz_learner* t, const dz_learner_config& cfg) {
  t->um = nullptr;
  memset(&t->buf, 0, sizeof(t->buf));
  t->cfg = cfg;
  t->lay = make_layout(cfg, &t->po);
  t->d = make_dims(cfg);
  t->fc = fc_net(cfg, t->d);
  t->B = cfg.batch;
  return carve(t, nullptr);   // the learner's split counts, which the actor's fp32 GEMMs share
}

// Noise of ONE apply, in this order: adv1_in[feat] adv1_out[512] adv2_in[512] adv2_out[A*atoms] val1_in[feat]
// val1_out[512] val2_in[512] val2_out[atoms]; every vector starts on a 4-float boundary.  Offsets in floats.  Rainbow;
// the noisy dueling network with one atom; the noisy plain network has only the first four (fc1 in / out, head in /
// out; the value stream's offsets are then those of the next apply and never read).
struct NoiseLayout {
  int64_t stride;   // floats per apply
  int64_t a1i, a1o, a2i, a2o, v1i, v1o, v2i, v2o;
};
NoiseLayout noise_layout(const dz_learner_config& c, const Dims& d) {
  NoiseLayout n;
  int64_t end = 0;
  auto next = [&](int64_t len) { const int64_t at = end; end += (len + 3) / 4 * 4; return at; };
  const int64_t atoms = c.kind == DZ_RAINBOW ? c.num_atoms : 1;
  n.a1i = next(d.feat); n.a1o = next(512); n.a2i = next(512); n.a2o = next((int64_t)c.num_actions * atoms);
  const int64_t one = end;
  n.v1i = next(d.feat); n.v1o = next(512); n.v2i = next(512); n.v2o = next(atoms);
  n.stride = two_streams(c) ? end : one;
  return n;
}
struct NoiseVecs { const float *a1i, *a1o, *a2i, *a2o, *v1i, *v1o, *v2i, *v2o; };
NoiseVecs noise_of(const dz_learner_config& c, const Dims& d, const float* base, int apply) {
  const NoiseLayout n = noise_layout(c, d);
  const float* p = base + (int64_t)apply * n.stride;
  return NoiseVecs{p + n.a1i, p + n.a1o, p + n.a2i, p + n.a2o, p + n.v1i, p + n.v1o, p + n.v2i, p + n.v2o};
}

UmNetDesc make_um_desc(const dz_learner* l) {
  const dz_learner_config& c = l->cfg;
  const Dims& d = l->d;
  const ParamOffsets& o = l->po;
  UmNetDesc u;
  memset(&u, 0, sizeof(u));
  const bool online_st = online_applies_to_s_t(c.kind);
  u.B = c.batch; u.H = d.H; u.W = d.W;
  const bool target_stm1 = is_munchausen(c.kind);   // online(s_tm1) | target(s_tm1) | target(s_t)
  u.npass = online_st || target_stm1 ? 3 : 2;
  u.pass_target[0] = 0; u.pass_target[1] = online_st ? 0 : 1; u.pass_target[2] = 1;
  u.online = l->buf.d_online; u.target = l->buf.d_target;
  for (int i = 0; i < 3; ++i) { u.off_conv_w[i] = o.conv_w[i]; u.off_conv_b[i] = o.conv_b[i]; }
  u.use_fc = !uses_iqn_net(c.kind);
  u.nstream = two_streams(c) ? 2 : 1;
  u.noisy = noisy_net(c) ? 1 : 0;
  if (u.use_fc)
    for (int s = 0; s < u.nstream; ++s) { u.off_fc_w[s] = o.w1[s]; u.off_fc_b[s] = o.b1[s]; }
  if (u.noisy) {
    const NoiseLayout nl = noise_layout(c, d);
    const int64_t in[2] = {nl.a1i, nl.v1i}, out[2] = {nl.a1o, nl.v1o};
    for (int s = 0; s < u.nstream; ++s) {
      u.off_fc_sw[s] = o.sw1[s]; u.off_fc_sb[s] = o.sb1[s];
      u.noise_off_in[s] = in[s]; u.noise_off_out[s] = out[s];
    }
    u.noise_stride = nl.stride;
    // apply p is noise slot p: online(s_tm1) | the middle pass | target(s_t); dqn's two passes read slots 0 and 2
    for (int p = 0; p < 3; ++p) u.noise_apply[p] = u.npass == 2 && p == 1 ? 2 : p;
  }
  return u;
}

GemmProblem zero_problem() {
  GemmProblem p;
  memset(&p, 0, sizeof(p));
  p.splits = 1;
  p.mul_div = 1;
  p.fd_per = make_fastdiv(1); p.fd_ow = make_fastdiv(1); p.fd_seg = make_fastdiv(1);
  return p;
}

void set_conv(GemmProblem& p, int mode, const void* A, int nimg, int H, int W, int Cin, int KH, int KW, int S) {
  p.a_mode = mode; p.A = A; p.H = H; p.W = W; p.Cin = Cin; p.KW = KW; p.S = S;
  p.OH = conv_out(H, KH, S); p.OW = conv_out(W, KW, S);
  p.seg = KW * Cin;
  p.fd_per = make_fastdiv(p.OH * p.OW); p.fd_ow = make_fastdiv(p.OW); p.fd_seg = make_fastdiv(p.seg);
  p.M = nimg * p.OH * p.OW;
  p.K = KH * KW * Cin;
}

template <typename KernelT>
int launch_batch(const char* tag, KernelT kernel, const GemmBatch& gb, dim3 grid, int threads, void* stream) {
  DZ_LAUNCH_NAMED(tag, kernel, grid, threads, 0, stream, gb);
  return DZ_OK;
}

// ---- NN launch helpers (tile shapes chosen by M / N) -------------------------------------------

int run_nn(const char* tag, GemmBatch& gb, bool dual, void* stream) {
  int maxM = 0, maxN = 0, maxS = 1;
  for (int i = 0; i < gb.n; ++i) {
    maxM = gb.p[i].M > maxM ? gb.p[i].M : maxM;
    maxN = gb.p[i].N > maxN ? gb.p[i].N : maxN;
    maxS = gb.p[i].splits > maxS ? gb.p[i].splits : maxS;
  }
  if (maxM <= 32) {
    dim3 grid((unsigned)ceil_div(maxN, 64), (unsigned)(ceil_div(maxM, 32) * maxS), gb.n);
    if (dual) return launch_batch(tag, gemm_nn_kernel<32, 64, 16, 2, 4, true>, gb, grid, 256, stream);
    return launch_batch(tag, gemm_nn_kernel<32, 64, 16, 2, 4, false>, gb, grid, 256, stream);
  }
  if (maxN <= 32 && !dual) {
    dim3 grid(1, (unsigned)(ceil_div(maxM, 64) * maxS), gb.n);
    return launch_batch(tag, gemm_nn_kernel<64, 32, 16, 4, 4, false>, gb, grid, 128, stream);
  }
  dim3 grid((unsigned)ceil_div(maxN, 64), (unsigned)(ceil_div(maxM, 64) * maxS), gb.n);
  if (dual) return launch_batch(tag, gemm_nn_kernel<64, 64, 16, 4, 4, true>, gb, grid, 256, stream);
  return launch_batch(tag, gemm_nn_kernel<64, 64, 16, 4, 4, false>, gb, grid, 256, stream);
}

int run_tn(const char* tag, GemmBatch& gb, void* stream) {
  int maxK = 0, maxN = 0, maxS = 1;
  for (int i = 0; i < gb.n; ++i) {
    int kext = gb.p[i].K + ((gb.p[i].Cb || gb.p[i].Cb2) ? 1 : 0);
    maxK = kext > maxK ? kext : maxK;
    maxN = gb.p[i].N > maxN ? gb.p[i].N : maxN;
    maxS = gb.p[i].splits > maxS ? gb.p[i].splits : maxS;
  }
  if (maxN <= 32) {
    dim3 grid(1, (unsigned)(ceil_div(maxK, 64) * maxS), gb.n);
    return launch_batch(tag, gemm_tn_kernel<64, 32, 16, 4, 2>, gb, grid, 256, stream);
  }
  dim3 grid((unsigned)ceil_div(maxN, 64), (unsigned)(ceil_div(maxK, 64) * maxS), gb.n);
  return launch_batch(tag, gemm_tn_kernel<64, 64, 16, 4, 4>, gb, grid, 256, stream);
}

int run_nt(const char* tag, GemmBatch& gb, bool dual, void* stream) {
  int maxM = 0, maxK = 0, maxS = 1;
  for (int i = 0; i < gb.n; ++i) {
    maxM = gb.p[i].M > maxM ? gb.p[i].M : maxM;
    maxK = gb.p[i].K > maxK ? gb.p[i].K : maxK;
    maxS = gb.p[i].splits > maxS ? gb.p[i].splits : maxS;
  }
  if (maxM <= 32) {
    dim3 grid((unsigned)ceil_div(maxK, 64), (unsigned)(ceil_div(maxM, 32) * maxS), gb.n);
    if (dual) return launch_batch(tag, gemm_nt_kernel<32, 64, 16, 2, 4, true>, gb, grid, 256, stream);
    return launch_batch(tag, gemm_nt_kernel<32, 64, 16, 2, 4, false>, gb, grid, 256, stream);
  }
  dim3 grid((unsigned)ceil_div(maxK, 64), (unsigned)(ceil_div(maxM, 64) * maxS), gb.n);
  if (dual) return launch_batch(tag, gemm_nt_kernel<64, 64, 16, 4, 4, true>, gb, grid, 256, stream);
  return launch_batch(tag, gemm_nt_kernel<64, 64, 16, 4, 4, false>, gb, grid, 256, stream);
}

// One noise apply per row of a noisy layer (rows of a batched-acting tick): same launch shape as run_nn's M <= 32 case,
// tiles of 32 rows.  noise_ld: floats between the noise applies of consecutive rows.
int run_nn_rownoise(const char* tag, GemmBatch& gb, long long noise_ld, void* stream) {
  int maxM = 0, maxN = 0, maxS = 1;
  for (int i = 0; i < gb.n; ++i) {
    if (gb.p[i].a_mode != A_PLAIN || !gb.p[i].B2 || !gb.p[i].a_scale || !gb.p[i].c_scale)
      return fail(DZ_EINVAL, "%s: per-row noise needs a plain noisy problem", tag);
    maxM = gb.p[i].M > maxM ? gb.p[i].M : maxM;
    maxN = gb.p[i].N > maxN ? gb.p[i].N : maxN;
    maxS = gb.p[i].splits > maxS ? gb.p[i].splits : maxS;
  }
  dim3 grid((unsigned)ceil_div(maxN, 64), (unsigned)(ceil_div(maxM, 32) * maxS), gb.n);
  DZ_LAUNCH_NAMED(tag, (gemm_nn_rownoise_kernel<32, 64, 16, 2, 4>), grid, 256, 0, stream, gb, noise_ld);
  return DZ_OK;
}

int finish_nn(const GemmBatch& gb, float* const* outs, bool dual, void* stream, long long noise_ld = 0) {
  FinishNNBatch fb;
  fb.n = gb.n;
  long long mx = 0;
  for (int i = 0; i < gb.n; ++i) {
    const GemmProblem& p = gb.p[i];
    fb.f[i] = FinishNN{p.C, p.splits, p.split_stride, p.M, p.N, dual ? 1 : 0, p.bias, p.bias2, p.c_scale, p.relu, p.bias_shared, outs[i]};
    long long t = (long long)p.M * p.N;
    mx = t > mx ? t : mx;
  }
  dim3 grid((unsigned)std::min<long long>(ceil_div(mx, 256), kNumSMs * 8), gb.n);   // grid-stride kernels
  if (noise_ld) DZ_LAUNCH(finish_nn_rownoise_kernel, grid, 256, 0, stream, fb, noise_ld);
  else DZ_LAUNCH(finish_nn_kernel, grid, 256, 0, stream, fb);
  return DZ_OK;
}

struct Pass {        // one network.apply
  const float* params;     // online or target blob
  int set;                 // torso activation set index (0..2)
  int head;                // head pass index (0..2)
  int apply;               // noise apply index (noisy layers): the step's slot 0 / 1 / 2
};

// ---- forward -----------------------------------------------------------------------------------

// The buffers a forward pass writes: torso activation sets [set], head outputs [head pass] (indices as in Pass), and
// the split-K partials of the fp32-FMA GEMMs.  The learner passes its own; an actor passes buffers sized for its streams.
struct NetBufs {
  float *act1[3], *act2[3], *act3[3];
  float *h1[3][2], *out[3], *outv[3];
  float *cosf[3], *hi[3];
  float* nn_partial;
  float* conv_partial;
  int split_rows;      // the fp32 fc1 / head GEMMs split K (into nn_partial) when the pass has at most this many images
};

NetBufs learner_bufs(const dz_learner* l) {
  NetBufs b;
  for (int p = 0; p < 3; ++p) {
    b.act1[p] = l->act1[p]; b.act2[p] = l->act2[p]; b.act3[p] = l->act3[p];
    b.h1[p][0] = l->h1[p][0]; b.h1[p][1] = l->h1[p][1]; b.out[p] = l->out[p]; b.outv[p] = l->outv[p];
    b.cosf[p] = l->cosf[p]; b.hi[p] = l->hi[p];
  }
  b.nn_partial = l->nn_partial;
  b.conv_partial = l->conv_partial;
  b.split_rows = 32;
  return b;
}

struct TorsoJob { const float* params; const uint8_t* const* rows; int set; };

int forward_torso(dz_learner* l, const NetBufs& nb, const TorsoJob* jobs, int njobs, int nimg, void* stream) {
  const Dims& d = l->d;
  const ParamOffsets& o = l->po;
  GemmBatch gb;
  gb.n = njobs;
  // conv1: uint8 rows gathered in place (K1 + K2 of SURVEY §2.1).  Not split over K (= 256): measured before the H100
  // port, the extra finish launch ate the gain of 2 or 3 splits.
  for (int i = 0; i < njobs; ++i) {
    GemmProblem p = zero_problem();
    set_conv(p, A_CONV_U8, jobs[i].rows, nimg, d.H, d.W, d.C, 8, 8, 4);
    p.B = jobs[i].params + o.conv_w[0]; p.bias = jobs[i].params + o.conv_b[0];
    p.N = 32; p.ldb = 32; p.ldc = 32; p.relu = 1; p.C = nb.act1[jobs[i].set];
    gb.p[i] = p;
  }
  DZ_TRY(run_nn("conv1_fwd", gb, false, stream));
  // conv2 / conv3: few output tiles (41 / 25 per pass) -> split K four ways so the grid covers the 132 SMs;
  // finish_nn adds the bias and ReLU.
  for (int layer = 2; layer <= 3; ++layer) {
    float* outs[kMaxProblems];
    for (int i = 0; i < njobs; ++i) {
      GemmProblem p = zero_problem();
      if (layer == 2) {
        set_conv(p, A_CONV_F32, nb.act1[jobs[i].set], nimg, d.h1, d.w1, 32, 4, 4, 2);
        p.B = jobs[i].params + o.conv_w[1]; p.bias = jobs[i].params + o.conv_b[1];
        outs[i] = nb.act2[jobs[i].set];
      } else {
        set_conv(p, A_CONV_F32, nb.act2[jobs[i].set], nimg, d.h2, d.w2, 64, 3, 3, 1);
        p.B = jobs[i].params + o.conv_w[2]; p.bias = jobs[i].params + o.conv_b[2];
        outs[i] = nb.act3[jobs[i].set];
      }
      p.N = 64; p.ldb = 64; p.ldc = 64; p.relu = 1;
      p.splits = l->conv_splits; p.split_stride = (long long)p.M * 64;
      p.C = nb.conv_partial + (long long)i * p.splits * p.split_stride;
      gb.p[i] = p;
    }
    DZ_TRY(run_nn(layer == 2 ? "conv2_fwd" : "conv3_fwd", gb, false, stream));
    DZ_TRY(finish_nn(gb, outs, false, stream));
  }
  return DZ_OK;
}

// The dueling head of `np` passes over `rows` rows: dueling_head_fwd_kernel, or for the noisy dueling network
// noisy_dueling_head_fwd_kernel.  Pass i reads h1[i][0] / h1[i][1] (advantage / value stream [rows][512]) and the head
// of params[i], and writes q [rows][A] to out[i]; noisy: through noise apply noise[i], or with noise_ld > 0 row r's
// apply at noise[i] + r * noise_ld.  The learner's forwards and dz_test_dueling_head_fwd run this function.
int launch_dueling_head_fwd(const dz_learner* l, int rows, int np, const float* const (*h1)[2], const float* const* params,
                            float* const* out, const float* const* noise, long long noise_ld, void* stream) {
  const ParamOffsets& o = l->po;
  const dz_learner_config& c = l->cfg;
  NoisyDuelingFwdArgs a;
  memset(&a, 0, sizeof(a));
  for (int i = 0; i < np; ++i) {
    a.h.h1[i][0] = h1[i][0]; a.h.h1[i][1] = h1[i][1];
    a.h.params[i] = params[i]; a.h.out[i] = out[i];
  }
  for (int s = 0; s < 2; ++s) { a.h.off_w[s] = o.w2[s]; a.h.off_b[s] = o.b2[s]; }
  a.h.rows = rows; a.h.A = c.num_actions;
  const dim3 grid((unsigned)ceil_div(rows, 8), (unsigned)np);
  if (!noisy_net(c)) {
    DZ_LAUNCH_NAMED("dueling_head_fwd", dueling_head_fwd_kernel, grid, 256, 0, stream, a.h);
    return DZ_OK;
  }
  const NoiseLayout nl = noise_layout(c, l->d);
  for (int i = 0; i < np; ++i) a.noise[i] = noise[i];
  for (int s = 0; s < 2; ++s) { a.off_sw[s] = o.sw2[s]; a.off_sb[s] = o.sb2[s]; }
  a.off_in[0] = nl.a2i; a.off_out[0] = nl.a2o; a.off_in[1] = nl.v2i; a.off_out[1] = nl.v2o;
  a.noise_ld = noise_ld;
  DZ_LAUNCH_NAMED("noisy_dueling_head_fwd", noisy_dueling_head_fwd_kernel, grid, 256, 0, stream, a);
  return DZ_OK;
}

// The dueling head's backward over `rows` rows of online(s_tm1): dueling_head_bwd_kernel, or for the noisy dueling
// network noisy_dueling_head_bwd_kernel through noise apply `noise`.  dq [rows][A] becomes dadv in place, dval [rows]
// is written, and both streams' dh1 [rows][512] from the head of `params`, masked by h1 > 0; with hi / lo (NULL: none)
// also their tf32 hi/lo pair.  The learner's backwards and dz_test_dueling_head_bwd run this function.
int launch_dueling_head_bwd(const dz_learner* l, int rows, float* dq, float* dval, const float* const* h1, const float* params,
                            float* const* dh1, float* const* hi, float* const* lo, const float* noise, void* stream) {
  const ParamOffsets& o = l->po;
  const dz_learner_config& c = l->cfg;
  NoisyDuelingBwdArgs a;
  memset(&a, 0, sizeof(a));
  a.g.dq = dq; a.g.dval = dval; a.g.B = rows; a.g.A = c.num_actions;
  for (int s = 0; s < 2; ++s) {
    a.g.h1[s] = h1[s]; a.g.W[s] = params + o.w2[s]; a.g.dh1[s] = dh1[s];
    if (hi) { a.g.hi[s] = hi[s]; a.g.lo[s] = lo[s]; }
  }
  if (!noisy_net(c)) {
    DZ_LAUNCH_NAMED("dueling_head_bwd", dueling_head_bwd_kernel, (unsigned)ceil_div(rows, 8), 256, 0, stream, a.g);
    return DZ_OK;
  }
  const NoiseVecs nz = noise_of(c, l->d, noise, 0);
  for (int s = 0; s < 2; ++s) a.S[s] = params + o.sw2[s];
  a.ein[0] = nz.a2i; a.eout[0] = nz.a2o; a.ein[1] = nz.v2i; a.eout[1] = nz.v2o;
  DZ_LAUNCH_NAMED("noisy_dueling_head_bwd", noisy_dueling_head_bwd_kernel, (unsigned)ceil_div(rows, 8), 256, 0, stream, a);
  return DZ_OK;
}

// Rainbow's noisy head of `np` passes over `nimg` <= kNhRows images in one launch (noisy_head_fwd_kernel): the passes
// that apply one parameter blob form a group, at most two passes each.  Pass i reads nb.h1[passes[i].head] and noise
// apply passes[i].apply, and writes nb.out / nb.outv of its head pass.  The learner step and dz_test_noisy_head_fwd
// run this function.
int launch_noisy_head_fwd(const dz_learner* l, const NetBufs& nb, const Pass* passes, int np, int nimg, const float* noise,
                          void* stream) {
  const ParamOffsets& o = l->po;
  const FcNet& f = l->fc;
  if (f.ns != 2 || !f.noisy || f.dueling_head || nimg < 1 || nimg > kNhRows)
    return fail(DZ_EINVAL, "noisy head: a two-stream noisy GEMM head over 1..32 images");
  NoisyHeadFwdArgs a;
  memset(&a, 0, sizeof(a));
  const float* blob[2] = {nullptr, nullptr};
  int ng = 0;
  for (int i = 0; i < np; ++i) {
    int g = 0;
    while (g < ng && !(blob[g] == passes[i].params && a.members[g] < 2)) ++g;
    if (g == 2) return fail(DZ_EINVAL, "noisy head: more than two groups of passes");
    if (g == ng) { blob[ng++] = passes[i].params; }
    const int q = a.members[g]++;
    const NoiseVecs nz = noise_of(l->cfg, l->d, noise, passes[i].apply);
    const int hp = passes[i].head;
    for (int s = 0; s < 2; ++s) {
      a.x[g][q][s] = nb.h1[hp][s];
      if ((reinterpret_cast<uintptr_t>(a.x[g][q][s]) & 15) != 0) return fail(DZ_EINVAL, "noisy head: h1 not 16-byte aligned");
      a.out[g][q][s] = s == 0 ? nb.out[hp] : nb.outv[hp];
      a.ein[g][q][s] = s == 0 ? nz.a2i : nz.v2i;
      a.eout[g][q][s] = s == 0 ? nz.a2o : nz.v2o;
    }
  }
  for (int g = 0; g < ng; ++g)
    for (int s = 0; s < 2; ++s) {
      a.mu[g][s] = blob[g] + o.w2[s]; a.sigma[g][s] = blob[g] + o.sw2[s];
      a.bias[g][s] = o.b2[s] < 0 ? nullptr : blob[g] + o.b2[s]; a.sbias[g][s] = blob[g] + o.sb2[s];
    }
  a.N[0] = (int)f.out[0]; a.N[1] = (int)f.out[1];
  a.tiles0 = (int)ceil_div(a.N[0], kNhTile);
  a.rows = nimg; a.bias_shared = f.shared_bias ? 1 : 0;
  DZ_CUDA_OK(cudaFuncSetAttribute(noisy_head_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kNhFwdSmem));
  const dim3 grid((unsigned)(a.tiles0 + ceil_div(a.N[1], kNhTile)), (unsigned)ng);
  DZ_LAUNCH_NAMED("noisy2_fwd", noisy_head_fwd_kernel, grid, 256, kNhFwdSmem, stream, a);
  return DZ_OK;
}

// Dynamic shared memory of noisy_head_bwd_kernel at B rows: every row of dout and the CTA's formed weights.
size_t noisy_head_bwd_smem(const FcNet& f, int B) { return (size_t)(B + kNhKc) * (f.out[0] + f.out[1]) * sizeof(float); }

// Rainbow's head input gradient through online(s_tm1) (noisy_head_bwd_kernel): dh1 of both streams from dout / doutv,
// and with hi / lo set their tf32 hi/lo pairs.  backward_fc and dz_test_noisy_head_bwd run this function.
int launch_noisy_head_bwd(const dz_learner* l, int B, const float* const* dout, const float* params, const float* noise,
                          const float* const* h1, float* const* dh1, float* const* hi, float* const* lo, void* stream) {
  const ParamOffsets& o = l->po;
  const FcNet& f = l->fc;
  if (f.ns != 2 || !f.noisy || f.dueling_head || B < 1 || B > kNhRows)
    return fail(DZ_EINVAL, "noisy head: a two-stream noisy GEMM head over 1..32 images");
  const NoiseVecs nz = noise_of(l->cfg, l->d, noise, 0);
  NoisyHeadBwdArgs a;
  memset(&a, 0, sizeof(a));
  for (int s = 0; s < 2; ++s) {
    a.dout[s] = dout[s]; a.mu[s] = params + o.w2[s]; a.sigma[s] = params + o.sw2[s];
    a.h1[s] = h1[s]; a.dh1[s] = dh1[s]; a.hi[s] = hi[s]; a.lo[s] = lo[s];
    a.N[s] = (int)f.out[s];
  }
  a.ein[0] = nz.a2i; a.eout[0] = nz.a2o; a.ein[1] = nz.v2i; a.eout[1] = nz.v2o;
  a.B = B;
  const size_t smem = noisy_head_bwd_smem(f, B);
  if (smem > kMaxDynSmem) return fail(DZ_EINVAL, "noisy head: the input gradient needs more than 227 KB of shared memory");
  if (smem > 48 * 1024)
    DZ_CUDA_OK(cudaFuncSetAttribute(noisy_head_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  DZ_LAUNCH_NAMED("noisy2_dgrad", noisy_head_bwd_kernel, (unsigned)(512 / kNhKc), 256, smem, stream, a);
  return DZ_OK;
}

// The layers after the torso (FcNet) of `np` passes over `nimg` images: rainbow's and the noisy networks' noisy layers
// (networks.py:137-178, DESIGN.md §17), the dueling network's streams (§16) and the plain network.  The 3136 -> 512
// layers of every pass and stream are one grouped launch (skipped with fc1_done: the tensor-core plan wrote h1), then
// the heads are one dueling head launch or one grouped launch; both GEMM stages split K into nn_partial when the pass
// has at most split_rows images.  Noisy layers read noise apply passes[i].apply of `noise`; with noise_ld > 0 (one pass
// only) image m uses its own apply at noise + m * noise_ld.  With noisy_head, rainbow's head of at most kNhRows images
// per pass is one launch_noisy_head_fwd instead (the learner step; acting keeps the grouped launch).
int forward_heads_fc(dz_learner* l, const NetBufs& nb, const Pass* passes, int np, int nimg, const float* noise, void* stream,
                     bool fc1_done = false, long long noise_ld = 0, bool noisy_head = false) {
  const Dims& d = l->d;
  const ParamOffsets& o = l->po;
  const dz_learner_config& c = l->cfg;
  const FcNet& f = l->fc;
  const int ns = f.ns;
  const int halves = f.noisy ? 2 : 1;   // a noisy problem's split partials carry a second (sigma) half
  if (ns * np > kMaxProblems) return fail(DZ_EINVAL, "too many passes for one grouped launch");
  if (noise_ld && (np != 1 || fc1_done)) return fail(DZ_EINVAL, "per-row noise: one pass with its own fc1");
  auto run = [&](const char* tag, GemmBatch& b) {
    return noise_ld ? run_nn_rownoise(tag, b, noise_ld, stream) : run_nn(tag, b, f.noisy, stream);
  };
  GemmBatch gb;
  gb.n = ns * np;
  float* outs[kMaxProblems];
  const int splits = nimg <= nb.split_rows ? l->fc_splits : 1;
  for (int i = 0; i < np && !fc1_done; ++i) {
    const float* prm = passes[i].params;
    const NoiseVecs nz = f.noisy ? noise_of(c, d, noise, passes[i].apply) : NoiseVecs{};
    for (int s = 0; s < ns; ++s) {
      GemmProblem p = zero_problem();
      p.a_mode = A_PLAIN; p.A = nb.act3[passes[i].set]; p.lda = d.feat; p.M = nimg; p.K = d.feat;
      p.B = prm + o.w1[s]; p.N = 512; p.ldb = 512; p.ldc = 512;
      p.bias = prm + o.b1[s]; p.relu = 1;
      if (f.noisy) {
        p.B2 = prm + o.sw1[s]; p.bias2 = prm + o.sb1[s];
        p.a_scale = s == 0 ? nz.a1i : nz.v1i; p.c_scale = s == 0 ? nz.a1o : nz.v1o;
      }
      const int q = ns * i + s;
      outs[q] = nb.h1[passes[i].head][s];
      if (splits > 1) {
        p.splits = splits; p.split_stride = (long long)halves * nimg * 512;
        p.C = nb.nn_partial + (long long)q * splits * p.split_stride;
      } else {
        p.C = outs[q];
      }
      gb.p[q] = p;
    }
  }
  if (!fc1_done) {
    DZ_TRY(run(f.noisy ? "noisy1_fwd" : "fc1_fwd", gb));
    if (splits > 1) DZ_TRY(finish_nn(gb, outs, f.noisy, stream, noise_ld));
  }
  if (f.dueling_head) {
    const float* h1[3][2];
    const float* prm[3];
    float* out[3];
    const float* noise_at[3];
    for (int i = 0; i < np; ++i) {
      const int hp = passes[i].head;
      h1[i][0] = nb.h1[hp][0]; h1[i][1] = nb.h1[hp][1];
      prm[i] = passes[i].params; out[i] = nb.out[hp];
      noise_at[i] = f.noisy ? noise + (int64_t)passes[i].apply * noise_layout(c, d).stride : nullptr;
    }
    return launch_dueling_head_fwd(l, nimg, np, h1, prm, out, noise_at, noise_ld, stream);
  }
  if (noisy_head && f.noisy && f.ns == 2 && !noise_ld && nimg <= kNhRows)
    return launch_noisy_head_fwd(l, nb, passes, np, nimg, noise, stream);
  const bool split_head = nimg <= nb.split_rows;
  for (int i = 0; i < np; ++i) {
    const float* prm = passes[i].params;
    const NoiseVecs nz = f.noisy ? noise_of(c, d, noise, passes[i].apply) : NoiseVecs{};
    for (int s = 0; s < ns; ++s) {
      const int n_out = (int)f.out[s];
      GemmProblem p = zero_problem();
      p.a_mode = A_PLAIN; p.A = nb.h1[passes[i].head][s]; p.lda = 512; p.M = nimg; p.K = 512;
      p.B = prm + o.w2[s]; p.N = n_out; p.ldb = n_out; p.ldc = n_out;
      p.bias = o.b2[s] < 0 ? nullptr : prm + o.b2[s]; p.bias_shared = f.shared_bias ? 1 : 0;
      if (f.noisy) {
        p.B2 = prm + o.sw2[s]; p.bias2 = prm + o.sb2[s];
        p.a_scale = s == 0 ? nz.a2i : nz.v2i; p.c_scale = s == 0 ? nz.a2o : nz.v2o;
      }
      const int q = ns * i + s;
      outs[q] = s == 0 ? nb.out[passes[i].head] : nb.outv[passes[i].head];
      if (split_head) {   // every problem's partials sized for the widest head, stream 0's
        p.splits = l->head_splits; p.split_stride = (long long)halves * nimg * n_out;
        p.C = nb.nn_partial + (long long)q * l->head_splits * halves * nimg * f.out[0];
      } else {
        p.C = outs[q];
      }
      gb.p[q] = p;
    }
  }
  DZ_TRY(run(f.noisy ? "noisy2_fwd" : "head_fwd", gb));
  if (split_head) DZ_TRY(finish_nn(gb, outs, f.noisy, stream, noise_ld));
  return DZ_OK;
}

// The cosine features out [rows][latent] of `rows` taus (iqn_cos_kernel).  forward_heads_iqn and dz_test_iqn_cos run
// this function.
int launch_iqn_cos(const float* taus, float* out, long long rows, int latent, void* stream) {
  DZ_LAUNCH(iqn_cos_kernel, (unsigned)ceil_div(rows * latent, 256), 256, 0, stream, taus, out, rows, latent);
  return DZ_OK;
}

// IQN's value head (iqn_head_fwd_kernel, A = num_actions <= kSkinnyMaxN) of `np` (<= 3) applies: apply i reads h1[i]
// [M[i]][512] and the head of params[i], and writes out[i] [M[i]][A].  forward_heads_iqn and dz_test_iqn_head_fwd run
// this function.
int launch_iqn_head_fwd(const dz_learner* l, int np, const float* const* h1, const float* const* params, float* const* out,
                        const int* M, void* stream) {
  const ParamOffsets& o = l->po;
  SkinnyHead h;
  memset(&h, 0, sizeof(h));
  h.n = np;
  int maxM = 0;
  for (int i = 0; i < np; ++i) {
    h.A[i] = h1[i]; h.W[i] = params[i] + o.w2[0]; h.bias[i] = params[i] + o.b2[0];
    h.out[i] = out[i]; h.M[i] = M[i];
    maxM = std::max(maxM, h.M[i]);
  }
  dim3 grid((unsigned)std::min<int64_t>(ceil_div(maxM, 8), kNumSMs * 2), (unsigned)np);
  DZ_LAUNCH_NAMED("iqn_head_fwd", iqn_head_fwd_kernel, grid, 256, 0, stream, h, l->d.out);
  return DZ_OK;
}

// The value head's input gradient dh1 [M][512] = [h1 > 0] dout W^T from dout [M][A] and the head of `params`
// (iqn_head_dgrad_kernel, A <= kSkinnyMaxN).  backward_iqn and dz_test_iqn_head_dgrad run this function.
int launch_iqn_head_dgrad(const dz_learner* l, const float* dout, const float* params, const float* h1, float* dh1, int M,
                          void* stream) {
  DZ_LAUNCH_NAMED("iqn_head_dgrad", iqn_head_dgrad_kernel, (unsigned)std::min<int64_t>(ceil_div((long long)M * 128, 256), kNumSMs * 8),
                  256, 0, stream, dout, params + l->po.w2[0], h1, dh1, M, l->d.out);
  return DZ_OK;
}

// The backward of E * F (E [B][N][D] the embedding after its ReLU, F [B][D] the state features): dfeat [B][D] and dE,
// in place in dhi (iqn_hadamard_bwd_kernel) or, packed, only as the transposed tf32 hi/lo image with rows k and
// reduction b * N + n (iqn_hadamard_bwd_packed_kernel: N == 64, D % 64 == 0; rg_total = the image's rows_pad / 8).
// backward_iqn and dz_test_iqn_hadamard_bwd run this function.
int launch_iqn_hadamard_bwd(bool packed, float* dhi, const float* E, const float* F, float* dfeat, float* img_hi, float* img_lo,
                            int rg_total, int B, int N, int D, void* stream) {
  if (packed) {
    dim3 hgrid((unsigned)(D / 64), (unsigned)B);
    DZ_LAUNCH(iqn_hadamard_bwd_packed_kernel, hgrid, 256, 0, stream, dhi, E, F, dfeat, img_hi, img_lo, rg_total, D);
  } else {
    DZ_LAUNCH(iqn_hadamard_bwd_kernel, (unsigned)ceil_div((long long)B * D, 256), 256, 0, stream, dhi, E, F, dfeat, B, N, D);
  }
  return DZ_OK;
}

// IQN embedding (latent -> 3136, ReLU, * state embedding) and 3136 -> 512 layer of the three network applies of
// one update on the packed-operand tensor-core kernels: one pack launch (cosine features + every weight operand of
// this step), the embedding GEMM whose epilogue writes the hi/lo tile images of the next GEMMs directly (the fp32
// `hi` tensors are never materialised), the split fc1 GEMM, one finish (bias + ReLU).
int iqn_embed_fc1_forward_packed(dz_learner* l, const NetBufs& nb, const Pass* passes, const GemmBatch& fc1, bool keep_E0, void* stream) {
  const Dims& d = l->d;
  const ParamOffsets& o = l->po;
  const dz_learner_config& c = l->cfg;
  PackBatch pb;
  memset(&pb, 0, sizeof(pb));
  const float* blob[2] = {nullptr, nullptr};   // distinct parameter blobs (online first)
  int widx[3];
  for (int i = 0; i < 3; ++i) {
    int k = 0;
    while (k < 2 && blob[k] && blob[k] != passes[i].params) ++k;
    if (k == 2) return fail(DZ_EINVAL, "iqn packed path expects at most two parameter blobs");
    blob[k] = passes[i].params; widx[i] = k;
    int hp = passes[i].head;
    const dz_learner::PkImg& im = l->pk_cos[hp];
    DZ_TRY(pk_add_job(pb, nb.cosf[hp], c.latent_dim, 1, fc1.p[i].M, c.latent_dim, im.rows_pad, im.red_pad, -1, im.hi, im.lo));
  }
  for (int k = 0; k < 2; ++k) {
    if (!blob[k]) continue;
    DZ_TRY(pk_add_job(pb, blob[k] + o.embed_w, d.feat, 0, d.feat, c.latent_dim, l->pk_weT[k].rows_pad, l->pk_weT[k].red_pad,
                      -1, l->pk_weT[k].hi, l->pk_weT[k].lo));
    DZ_TRY(pk_add_job(pb, blob[k] + o.w1[0], 512, 0, 512, d.feat, l->pk_wT[k].rows_pad, l->pk_wT[k].red_pad, -1,
                      l->pk_wT[k].hi, l->pk_wT[k].lo));
  }
  // backward-time operand that only depends on forward-time tensors: W (rows k, reduction n) for the input gradient
  DZ_TRY(pk_add_job(pb, l->buf.d_online + o.w1[0], 512, 1, d.feat, 512, l->pk_w.rows_pad, l->pk_w.red_pad, -1, l->pk_w.hi, l->pk_w.lo));
  DZ_TRY(launch_pack("iqn_pack_fwd", pb, stream));

  PkBatch eb;
  memset(&eb, 0, sizeof(eb));
  eb.n = 3;
  for (int i = 0; i < 3; ++i) {
    int hp = passes[i].head;
    const bool keep = keep_E0 && hp == 0;
    const dz_learner::PkImg &cs = l->pk_cos[hp], &we = l->pk_weT[widx[i]], &im = l->pk_act[hp];
    const PkTarget img{im.hi, im.lo, im.rows_pad / 8};
    const PkTarget imgT = keep ? PkTarget{l->pk_actT.hi, l->pk_actT.lo, l->pk_actT.rows_pad / 8} : PkTarget{nullptr, nullptr, 0};
    eb.p[i] = pk_embed_problem(PkOperand{cs.hi, cs.lo, cs.rows_pad / 8}, PkOperand{we.hi, we.lo, we.rows_pad / 8}, fc1.p[i].M,
                               d.feat, cs.red_pad / kPkKB, passes[i].params + o.embed_b, nb.act3[passes[i].set], l->n_head[hp],
                               d.feat, keep ? l->E0 : nullptr, img, imgT);
  }
  DZ_TRY(launch_pgemm("iqn_embed_fwd", eb, stream, 1));

  PkBatch kb;
  memset(&kb, 0, sizeof(kb));
  kb.n = 3;
  GemmBatch fin = fc1;
  float* outs[kMaxProblems] = {nullptr};
  long long off = 0;
  for (int i = 0; i < 3; ++i) {
    int hp = passes[i].head;
    const dz_learner::PkImg& im = l->pk_act[hp];
    PkProblem& p = kb.p[i];
    p.A = PkOperand{im.hi, im.lo, im.rows_pad / 8};
    p.B = PkOperand{l->pk_wT[widx[i]].hi, l->pk_wT[widx[i]].lo, l->pk_wT[widx[i]].rows_pad / 8};
    p.MI = fc1.p[i].M; p.NJ = 512; p.nkb = im.red_pad / kPkKB;
    p.sc_i = 512; p.sc_j = 1; p.splits = l->pk_fwd_splits;
    p.split_stride = (long long)p.MI * 512;
    p.C = l->pk_fwd_partial + off;
    off += (long long)p.splits * p.split_stride;
    p.bias_j = fc1.p[i].bias; p.relu = 1;
    if (p.splits == 1) p.C = fc1.p[i].C;
    fin.p[i].C = p.C; fin.p[i].splits = p.splits; fin.p[i].split_stride = p.split_stride;
    outs[i] = fc1.p[i].C;
  }
  DZ_TRY(launch_pgemm("iqn_fc1_fwd", kb, stream));
  if (l->pk_fwd_splits > 1) DZ_TRY(finish_nn(fin, outs, false, stream));
  return DZ_OK;
}

// IQN (networks.py:264-292): cosine embedding -> linear -> relu -> * state embedding -> value head.  `row_invariant`: the
// value head takes the one-warp-per-row kernel at any row count (where the head is narrow enough), so that a row's
// bits do not depend on how many rows the call holds (fqf's acting; the fp32 GEMMs before it never split K here).
int forward_heads_iqn(dz_learner* l, const NetBufs& nb, const Pass* passes, int np, int nimg, const float* const* taus, bool keep_E0, void* stream,
                      bool row_invariant = false) {
  const Dims& d = l->d;
  const ParamOffsets& o = l->po;
  const dz_learner_config& c = l->cfg;
  GemmBatch gb;
  gb.n = np;
  for (int i = 0; i < np; ++i)
    DZ_TRY(launch_iqn_cos(taus[i], nb.cosf[passes[i].head], (long long)nimg * l->n_head[passes[i].head], c.latent_dim, stream));
  const bool packed = l->pk_on && nimg == l->B && np == 3;
  if (!packed) {
    for (int i = 0; i < np; ++i) {
      int hp = passes[i].head;
      GemmProblem p = zero_problem();
      p.a_mode = A_PLAIN; p.A = nb.cosf[hp]; p.lda = c.latent_dim; p.M = nimg * l->n_head[hp]; p.K = c.latent_dim;
      p.B = passes[i].params + o.embed_w; p.N = d.feat; p.ldb = d.feat; p.ldc = d.feat;
      p.bias = passes[i].params + o.embed_b; p.relu = 1;
      p.mul = nb.act3[passes[i].set]; p.mul_div = l->n_head[hp];
      p.C = nb.hi[hp]; p.C2 = (keep_E0 && hp == 0) ? l->E0 : nullptr;
      gb.p[i] = p;
    }
    DZ_TRY(run_nn("iqn_embed_fwd", gb, false, stream));
  }
  for (int i = 0; i < np; ++i) {
    int hp = passes[i].head;
    GemmProblem p = zero_problem();
    p.a_mode = A_PLAIN; p.A = nb.hi[hp]; p.lda = d.feat; p.M = nimg * l->n_head[hp]; p.K = d.feat;
    p.B = passes[i].params + o.w1[0]; p.N = 512; p.ldb = 512; p.ldc = 512;
    p.bias = passes[i].params + o.b1[0]; p.relu = 1; p.C = nb.h1[hp][0];
    gb.p[i] = p;
  }
  // M can be small when acting (1 x tau_samples_policy rows): same kernel family handles it
  if (packed) {
    DZ_TRY(iqn_embed_fc1_forward_packed(l, nb, passes, gb, keep_E0, stream));
  } else {
    DZ_TRY(run_nn("iqn_fc1_fwd", gb, false, stream));
  }
  if (((long long)nimg * l->n_head[passes[0].head] >= 512 || row_invariant) && d.out <= kSkinnyMaxN && np <= 3) {
    const float* h1[3];
    const float* prm[3];
    float* out[3];
    int M[3];
    for (int i = 0; i < np; ++i) {
      int hp = passes[i].head;
      h1[i] = nb.h1[hp][0]; prm[i] = passes[i].params; out[i] = nb.out[hp]; M[i] = nimg * l->n_head[hp];
    }
    return launch_iqn_head_fwd(l, np, h1, prm, out, M, stream);
  }
  for (int i = 0; i < np; ++i) {
    int hp = passes[i].head;
    GemmProblem p = zero_problem();
    p.a_mode = A_PLAIN; p.A = nb.h1[hp][0]; p.lda = 512; p.M = nimg * l->n_head[hp]; p.K = 512;
    p.B = passes[i].params + o.w2[0]; p.N = d.out; p.ldb = d.out; p.ldc = d.out;
    p.bias = passes[i].params + o.b2[0]; p.C = nb.out[hp];
    gb.p[i] = p;
  }
  DZ_TRY(run_nn("iqn_head_fwd", gb, false, stream));
  return DZ_OK;
}

// ---- backward ----------------------------------------------------------------------------------

FinishNT make_finish_nt(const GemmProblem* probs, int nsrc, const float* mask, float* out, bool dual, float* out_hi = nullptr,
                        float* out_lo = nullptr) {
  FinishNT f;
  memset(&f, 0, sizeof(f));
  f.nsrc = nsrc; f.splits = probs[0].splits; f.stride = probs[0].split_stride; f.M = probs[0].M; f.K = probs[0].K;
  f.dual = dual ? 1 : 0; f.mask = mask; f.out = out; f.out_hi = out_hi; f.out_lo = out_lo;
  for (int q = 0; q < nsrc; ++q) { f.partial[q] = probs[q].C; f.a_scale[q] = probs[q].a_scale; }
  return f;
}
int finish_nt_batch(const FinishNT* jobs, int njobs, void* stream) {
  FinishNTBatch fb;
  memset(&fb, 0, sizeof(fb));
  long long total = 0;
  for (int j = 0; j < njobs; ++j) { fb.f[j] = jobs[j]; total = std::max(total, (long long)jobs[j].M * jobs[j].K); }
  dim3 grid((unsigned)std::min<long long>(ceil_div(total, 256), kNumSMs * 8), (unsigned)njobs);
  DZ_LAUNCH(finish_nt_kernel, grid, 256, 0, stream, fb);
  return DZ_OK;
}
int finish_nt(const GemmProblem* probs, int nsrc, const float* mask, float* out, bool dual, void* stream) {
  FinishNT f = make_finish_nt(probs, nsrc, mask, out, dual);
  return finish_nt_batch(&f, 1, stream);
}

bool split_norm_active(const dz_learner* l);

// Torso backward from dact3 (already masked by act3 > 0): conv3/conv2/conv1 weight+bias grads.
int backward_torso(dz_learner* l, const uint8_t* const* rows0, void* stream) {
  const Dims& d = l->d;
  const ParamOffsets& o = l->po;
  const int B = l->B;
  float* G = l->buf.d_grads;
  const float* P = l->buf.d_online;
  FinishTNBatch fb;
  fb.n = 0;
  GemmBatch gb;
  if (l->um && uses_iqn_net(l->cfg.kind)) DZ_TRY(um_split_dact3(l->um, stream));   // dact3 came from the Hadamard kernel (fp32)
  // conv3 wgrad
  float* norm_parts = split_norm_active(l) ? l->norm_parts : nullptr;
  if (l->um) {   // conv3 weight gradient + its finish (partial sums, bias gradient, split-norm partials) on a side stream
    void* ws = l->side3.fork(stream, stream);
    DZ_TRY(um_wgrad_conv3(l->um, ws));
    DZ_TRY(um_wgrad_finish_layer(l->um, 3, G + o.conv_w[2], G + o.conv_b[2], norm_parts, ws));
  } else {
    GemmProblem p = zero_problem();
    set_conv(p, A_CONV_F32, l->act2[0], B, d.h2, d.w2, 64, 3, 3, 1);
    p.B = l->dact3; p.N = 64; p.ldb = 64; p.ldc = 64;
    p.Cb = G + o.conv_b[2];
    int splits = (int)std::min<int64_t>(32, ceil_div(p.M, 64));
    p.splits = splits; p.split_stride = (long long)(p.K + 1) * 64; p.C = l->tn_partial[2];
    gb.n = 1; gb.p[0] = p;
    DZ_TRY(run_tn("conv3_wgrad", gb, l->side.fork(stream, stream)));
    fb.f[fb.n++] = FinishTN{p.C, splits, p.split_stride, p.K, 64, G + o.conv_w[2], nullptr, p.Cb, nullptr, nullptr, nullptr};
  }
  // conv3 dgrad: dcol = dpre3 * W3^T ; col2im with ReLU mask of act2
  if (l->um) {
    DZ_TRY(um_backward_conv3(l->um, stream));
  } else {
    GemmProblem p = zero_problem();
    p.A = l->dact3; p.lda = 64; p.M = B * d.h3 * d.w3; p.N = 64; p.K = 576;
    p.B = P + o.conv_w[2]; p.ldb = 64; p.C = l->dcol; p.ldc = 576;
    gb.n = 1; gb.p[0] = p;
    DZ_TRY(run_nt("conv3_dgrad", gb, false, stream));
    long long total = (long long)B * d.h2 * d.w2 * 64;
    DZ_LAUNCH(col2im_kernel, (unsigned)ceil_div(total, 256), 256, 0, stream, l->dcol, l->act2[0], l->dact2, B, d.h2, d.w2, 64, 3, 3, 1,
              d.h3, d.w3);
  }
  // conv2 wgrad
  if (l->um) {   // conv2: on the second side stream, beside conv3's (both fit next to the input-gradient kernels)
    void* ws = l->side2.fork(stream, stream);
    DZ_TRY(um_wgrad_conv2(l->um, ws));
    DZ_TRY(um_wgrad_finish_layer(l->um, 2, G + o.conv_w[1], G + o.conv_b[1], norm_parts, ws));
  } else {
    GemmProblem p = zero_problem();
    set_conv(p, A_CONV_F32, l->act1[0], B, d.h1, d.w1, 32, 4, 4, 2);
    p.B = l->dact2; p.N = 64; p.ldb = 64; p.ldc = 64;
    p.Cb = G + o.conv_b[1];
    int splits = (int)std::min<int64_t>(32, ceil_div(p.M, 64));
    p.splits = splits; p.split_stride = (long long)(p.K + 1) * 64; p.C = l->tn_partial[1];
    gb.n = 1; gb.p[0] = p;
    DZ_TRY(run_tn("conv2_wgrad", gb, l->side.fork(stream, stream)));
    fb.f[fb.n++] = FinishTN{p.C, splits, p.split_stride, p.K, 64, G + o.conv_w[1], nullptr, p.Cb, nullptr, nullptr, nullptr};
  }
  // conv2 dgrad
  if (l->um) {
    DZ_TRY(um_backward_conv2(l->um, stream));
  } else {
    GemmProblem p = zero_problem();
    p.A = l->dact2; p.lda = 64; p.M = B * d.h2 * d.w2; p.N = 64; p.K = 512;
    p.B = P + o.conv_w[1]; p.ldb = 64; p.C = l->dcol; p.ldc = 512;
    gb.n = 1; gb.p[0] = p;
    DZ_TRY(run_nt("conv2_dgrad", gb, false, stream));
    long long total = (long long)B * d.h1 * d.w1 * 32;
    DZ_LAUNCH(col2im_kernel, (unsigned)ceil_div(total, 256), 256, 0, stream, l->dcol, l->act1[0], l->dact1, B, d.h1, d.w1, 32, 4, 4, 2,
              d.h2, d.w2);
  }
  // conv1 wgrad (A = uint8 rows in place)
  if (l->um) {
    void* ws = l->side3.fork(stream, stream);
    DZ_TRY(um_wgrad_conv1(l->um, rows0, ws));
    DZ_TRY(um_wgrad_finish_layer(l->um, 1, G + o.conv_w[0], G + o.conv_b[0], norm_parts, ws));
    DZ_TRY(l->side3.join(stream));
    DZ_TRY(l->side2.join(stream));
    return l->side.join(stream);
  } else {
    GemmProblem p = zero_problem();
    set_conv(p, A_CONV_U8, rows0, B, d.H, d.W, d.C, 8, 8, 4);
    p.B = l->dact1; p.N = 32; p.ldb = 32; p.ldc = 32;
    p.Cb = G + o.conv_b[0];
    int splits = (int)std::min<int64_t>(64, ceil_div(p.M, 64));
    p.splits = splits; p.split_stride = (long long)(p.K + 1) * 32; p.C = l->tn_partial[0];
    gb.n = 1; gb.p[0] = p;
    DZ_TRY(run_tn("conv1_wgrad", gb, l->side.fork(stream, stream)));
    fb.f[fb.n++] = FinishTN{p.C, splits, p.split_stride, p.K, 32, G + o.conv_w[0], nullptr, p.Cb, nullptr, nullptr, nullptr};
  }
  void* ws = l->side.tail(stream);   // after conv1_wgrad on the same (side) stream
  dim3 grid((unsigned)ceil_div(577 * 64, 256), fb.n);
  DZ_LAUNCH(finish_tn_kernel, grid, 256, 0, ws, fb);
  return l->side.join(stream);
}

// The backward of forward_heads_fc through online(s_tm1), noise apply 0 of `noise` for noisy layers: the dueling head
// kernel (dout -> dadv in place, dval -> doutv, both streams' dh1), the head and 3136 -> 512 weight gradients on the
// side stream (a noisy one fills the mu and sigma gradients together), the GEMM heads' input gradient, and dact3, which
// sums every stream's input gradient.  On the tensor-core path fc1's input gradient reads dh1 as a tf32 hi/lo pair,
// written by the dueling head kernel or by a split head input gradient's finish, else by um_split_dh1.
int backward_fc(dz_learner* l, const float* noise, void* stream) {
  const Dims& d = l->d;
  const ParamOffsets& o = l->po;
  const FcNet& f = l->fc;
  const int B = l->B, ns = f.ns;
  const int halves = f.noisy ? 2 : 1;   // a noisy problem's split partials carry a second (sigma) half
  float* G = l->buf.d_grads;
  const float* P = l->buf.d_online;
  const NoiseVecs nz = f.noisy ? noise_of(l->cfg, d, noise, 0) : NoiseVecs{};
  const float* in1[2] = {nz.a1i, nz.v1i};
  const float* out1[2] = {nz.a1o, nz.v1o};
  const float* in2[2] = {nz.a2i, nz.v2i};
  const float* out2[2] = {nz.a2o, nz.v2o};
  float* dout[2] = {l->dout, l->doutv};
  float* hi[2] = {nullptr, nullptr};
  float* lo[2] = {nullptr, nullptr};
  if (l->um)
    for (int s = 0; s < ns; ++s) { hi[s] = um_dh1_hi(l->um, s); lo[s] = um_dh1_lo(l->um, s); }
  bool hilo_done = false;
  if (f.dueling_head) {
    const float* h1[2] = {l->h1[0][0], l->h1[0][1]};
    DZ_TRY(launch_dueling_head_bwd(l, B, l->dout, l->doutv, h1, P, l->dh1, hi, lo, noise, stream));
    hilo_done = true;
  }
  GemmBatch gb;
  gb.n = ns;
  float* bias_terms = l->scalars + 8 + kNormBlocks;   // a shared bias: the per-output terms sum_to_scalar_kernel adds
  for (int s = 0; s < ns; ++s) {  // head weight and bias gradients
    const int n_out = (int)f.out[s];
    GemmProblem p = zero_problem();
    p.a_mode = A_PLAIN; p.A = l->h1[0][s]; p.lda = 512; p.M = B; p.K = 512;
    p.B = dout[s]; p.N = n_out; p.ldb = n_out; p.ldc = n_out;
    p.C = G + o.w2[s]; p.Cb = f.shared_bias ? bias_terms : o.b2[s] < 0 ? nullptr : G + o.b2[s];
    if (f.noisy) { p.C2 = G + o.sw2[s]; p.Cb2 = G + o.sb2[s]; p.a_scale = in2[s]; p.c_scale = out2[s]; }
    gb.p[s] = p;
  }
  DZ_TRY(run_tn(f.noisy ? "noisy2_wgrad" : "head_wgrad", gb, l->side.fork(stream, stream)));
  if (f.shared_bias) DZ_LAUNCH(sum_to_scalar_kernel, 1, 128, 0, l->side.tail(stream), bias_terms, d.out, G + o.b2[0]);
  // rainbow: one launch without split partials, when every row of dout fits in shared memory (not at the widest heads,
  // e.g. 64 actions x 128 atoms, which keep the split input gradient below)
  if (!f.dueling_head && f.noisy && ns == 2 && B <= kNhRows && noisy_head_bwd_smem(f, B) <= kMaxDynSmem) {
    const float* h1[2] = {l->h1[0][0], l->h1[0][1]};
    DZ_TRY(launch_noisy_head_bwd(l, B, dout, P, noise, h1, l->dh1, hi, lo, stream));
    hilo_done = true;
  } else if (!f.dueling_head) {  // dh1_s = dout_s * W2_s^T, masked by h1_s > 0
    // Noisy heads split the reduction 4 ways.  Wide plain heads (c51: 306 outputs, qr-dqn: 1206): with one CTA column
    // per 64 outputs of dh1 the reduction over the head width is a serial chain (measured 24 / 65 us); split it.  The
    // finish of the split partials applies the mask and, on the tensor-core path, writes the tf32 hi/lo pair, which
    // saves the separate split launch; unsplit, the GEMM applies the mask.
    const int splits = f.noisy ? 4 : d.out > 64 ? (int)std::min<int64_t>(16, ceil_div(d.out, 96)) : 1;
    for (int s = 0; s < ns; ++s) {
      const int n_out = (int)f.out[s];
      GemmProblem p = zero_problem();
      p.A = dout[s]; p.lda = n_out; p.M = B; p.N = n_out; p.K = 512;
      p.B = P + o.w2[s]; p.ldb = n_out; p.ldc = 512;
      if (f.noisy) { p.B2 = P + o.sw2[s]; p.a_scale = in2[s]; p.c_scale = out2[s]; }
      if (splits > 1) {
        p.splits = splits; p.split_stride = (long long)halves * B * 512;
        p.C = l->nt_partial + (long long)s * splits * p.split_stride;
      } else {
        p.C = l->dh1[s]; p.mask = l->h1[0][s];
      }
      gb.p[s] = p;
    }
    DZ_TRY(run_nt(f.noisy ? "noisy2_dgrad" : "head_dgrad", gb, f.noisy, stream));
    if (splits > 1) {   // every stream's dh1 in one launch
      FinishNT jobs[2];
      for (int s = 0; s < ns; ++s) jobs[s] = make_finish_nt(&gb.p[s], 1, l->h1[0][s], l->dh1[s], f.noisy, hi[s], lo[s]);
      DZ_TRY(finish_nt_batch(jobs, ns, stream));
      hilo_done = true;
    }
  }
  for (int s = 0; s < ns; ++s) {  // 3136 -> 512 weight and bias gradients
    GemmProblem p = zero_problem();
    p.a_mode = A_PLAIN; p.A = l->act3[0]; p.lda = d.feat; p.M = B; p.K = d.feat;
    p.B = l->dh1[s]; p.N = 512; p.ldb = 512; p.ldc = 512;
    p.C = G + o.w1[s]; p.Cb = G + o.b1[s];
    if (f.noisy) { p.C2 = G + o.sw1[s]; p.Cb2 = G + o.sb1[s]; p.a_scale = in1[s]; p.c_scale = out1[s]; }
    gb.p[s] = p;
  }
  DZ_TRY(run_tn(f.noisy ? "noisy1_wgrad" : "fc1_wgrad", gb, l->side.fork(stream, stream)));
  if (l->um) {   // dact3 on the tensor-core path: W streamed once through TMA, split partials + masked finish
    if (!hilo_done) DZ_TRY(um_split_dh1(l->um, stream));
    return um_backward_fc(l->um, f.noisy ? noise : nullptr, stream);
  }
  for (int s = 0; s < ns; ++s) {  // dact3 = (sum over streams of dh1_s * W1_s^T) * [act3 > 0]
    GemmProblem p = zero_problem();
    p.A = l->dh1[s]; p.lda = 512; p.M = B; p.N = 512; p.K = d.feat;
    p.B = P + o.w1[s]; p.ldb = 512; p.ldc = d.feat;
    if (f.noisy) { p.B2 = P + o.sw1[s]; p.a_scale = in1[s]; p.c_scale = out1[s]; }
    // weight-streaming GEMM with a 32-row output: split the reduction so ~400 CTAs keep HBM busy
    p.splits = l->nt_splits; p.split_stride = (long long)halves * B * d.feat;
    p.C = l->nt_partial + (long long)s * l->nt_splits * p.split_stride;
    gb.p[s] = p;
  }
  DZ_TRY(run_nt(f.noisy ? "noisy1_dgrad" : "fc1_dgrad", gb, f.noisy, stream));
  return finish_nt(gb.p, ns, l->act3[0], l->dact3, f.noisy, stream);
}

int backward_iqn(dz_learner* l, void* stream) {
  const Dims& d = l->d;
  const ParamOffsets& o = l->po;
  const dz_learner_config& c = l->cfg;
  const int B = l->B, N = l->n_head[0], M = B * N;
  float* G = l->buf.d_grads;
  const float* P = l->buf.d_online;
  GemmBatch gb;
  gb.n = 1;
  FinishTNBatch fb;
  fb.n = 0;
  float* part_head = l->tn_partial[3];
  float* part_embed = l->tn_partial[3] + (long long)16 * 513 * 64;
  {  // head wgrad: reduction over M rows
    GemmProblem p = zero_problem();
    p.a_mode = A_PLAIN; p.A = l->h1[0][0]; p.lda = 512; p.M = M; p.K = 512;
    p.B = l->dout; p.N = d.out; p.ldb = d.out; p.ldc = d.out;
    p.Cb = G + o.b2[0];
    int splits = (int)std::min<int64_t>(16, ceil_div(M, 64));
    p.splits = splits; p.split_stride = (long long)513 * d.out; p.C = part_head;
    gb.p[0] = p;
    DZ_TRY(run_tn("iqn_head_wgrad", gb, l->side.fork(stream, stream)));
    fb.f[fb.n++] = FinishTN{p.C, splits, p.split_stride, 512, d.out, G + o.w2[0], nullptr, p.Cb, nullptr, nullptr, nullptr};
  }
  {  // dh1
    GemmProblem p = zero_problem();
    p.A = l->dout; p.lda = d.out; p.M = M; p.N = d.out; p.K = 512;
    p.B = P + o.w2[0]; p.ldb = d.out; p.C = l->dh1[0]; p.ldc = 512; p.mask = l->h1[0][0];
    gb.p[0] = p;
    if (M >= 512 && d.out <= kSkinnyMaxN) {
      DZ_TRY(launch_iqn_head_dgrad(l, l->dout, P, l->h1[0][0], l->dh1[0], M, stream));
    } else {
      DZ_TRY(run_nt("iqn_head_dgrad", gb, false, stream));
    }
  }
  if (l->pk_on) {
    // dh1 in both operand orientations, then the two big contractions on the tensor-core kernel
    PackBatch pb;
    memset(&pb, 0, sizeof(pb));
    DZ_TRY(pk_add_job(pb, l->dh1[0], 512, 0, 512, M, l->pk_dh1T.rows_pad, l->pk_dh1T.red_pad, -1, l->pk_dh1T.hi, l->pk_dh1T.lo));
    DZ_TRY(pk_add_job(pb, l->dh1[0], 512, 1, M, 512, l->pk_dh1.rows_pad, l->pk_dh1.red_pad, -1, l->pk_dh1.hi, l->pk_dh1.lo));
    if (l->pk_embed_bwd)   // cos^T plus a row of ones (bias gradient) for the embedding weight gradient
      DZ_TRY(pk_add_job(pb, l->cosf[0], c.latent_dim, 0, c.latent_dim, M, l->pk_cosT.rows_pad, l->pk_cosT.red_pad, c.latent_dim,
                        l->pk_cosT.hi, l->pk_cosT.lo));
    DZ_TRY(launch_pack("iqn_fc1_pack_bwd", pb, stream));
    PkBatch kb;
    memset(&kb, 0, sizeof(kb));
    kb.n = 1;
    {  // fc1 wgrad: [feat + 1 (bias row), 512] = hi0^T(+ones) * dh1, reduction over the M rows, split partials
      PkProblem& p = kb.p[0];
      p.A = PkOperand{l->pk_actT.hi, l->pk_actT.lo, l->pk_actT.rows_pad / 8};
      p.B = PkOperand{l->pk_dh1T.hi, l->pk_dh1T.lo, l->pk_dh1T.rows_pad / 8};
      p.MI = d.feat + 1; p.NJ = 512; p.nkb = l->pk_actT.red_pad / kPkKB;
      p.sc_i = 512; p.sc_j = 1; p.splits = l->pk_wgrad_splits; p.split_stride = (long long)(d.feat + 1) * 512;
      p.C = l->pk_wgrad_partial;
      DZ_TRY(launch_pgemm("iqn_fc1_wgrad", kb, l->side.fork(stream, stream)));
      fb.f[fb.n++] = FinishTN{p.C, p.splits, p.split_stride, d.feat, 512, G + o.w1[0], nullptr, G + o.b1[0], nullptr, nullptr, nullptr};
    }
    {  // dHI[m,k] = sum_n dh1[m,n] W[k,n]
      PkProblem& p = kb.p[0];
      memset(&p, 0, sizeof(p));
      p.A = PkOperand{l->pk_dh1.hi, l->pk_dh1.lo, l->pk_dh1.rows_pad / 8};
      p.B = PkOperand{l->pk_w.hi, l->pk_w.lo, l->pk_w.rows_pad / 8};
      p.MI = M; p.NJ = d.feat; p.nkb = l->pk_dh1.red_pad / kPkKB;
      p.sc_i = d.feat; p.sc_j = 1; p.splits = 1; p.split_stride = 0; p.C = l->dhi;
      DZ_TRY(launch_pgemm("iqn_fc1_dgrad", kb, stream));
    }
  } else {
  {  // fc1 wgrad (reduction over M rows, no split: 400 tiles already)
    GemmProblem p = zero_problem();
    p.a_mode = A_PLAIN; p.A = l->hi[0]; p.lda = d.feat; p.M = M; p.K = d.feat;
    p.B = l->dh1[0]; p.N = 512; p.ldb = 512; p.ldc = 512;
    p.C = G + o.w1[0]; p.Cb = G + o.b1[0];
    gb.p[0] = p;
    DZ_TRY(run_tn("iqn_fc1_wgrad", gb, l->side.fork(stream, stream)));
  }
  {  // dHI = dh1 * Wf^T
    GemmProblem p = zero_problem();
    p.A = l->dh1[0]; p.lda = 512; p.M = M; p.N = 512; p.K = d.feat;
    p.B = P + o.w1[0]; p.ldb = 512; p.C = l->dhi; p.ldc = d.feat;
    gb.p[0] = p;
    DZ_TRY(run_nt("iqn_fc1_dgrad", gb, false, stream));
  }
  }
  if (l->pk_embed_bwd) {
    DZ_TRY(launch_iqn_hadamard_bwd(true, l->dhi, l->E0, l->act3[0], l->dact3, l->pk_dET.hi, l->pk_dET.lo, l->pk_dET.rows_pad / 8,
                                   B, N, d.feat, stream));
    // embed wgrad: [feat, latent + 1 (bias column)] = dE^T * [cos | 1], stored transposed into the [latent + 1, feat] partials
    PkBatch kb;
    memset(&kb, 0, sizeof(kb));
    kb.n = 1;
    PkProblem& p = kb.p[0];
    p.A = PkOperand{l->pk_dET.hi, l->pk_dET.lo, l->pk_dET.rows_pad / 8};
    p.B = PkOperand{l->pk_cosT.hi, l->pk_cosT.lo, l->pk_cosT.rows_pad / 8};
    p.MI = d.feat; p.NJ = c.latent_dim + 1; p.nkb = l->pk_dET.red_pad / kPkKB;
    p.sc_i = 1; p.sc_j = d.feat; p.splits = l->pk_embed_wgrad_splits; p.split_stride = (long long)(c.latent_dim + 1) * d.feat;
    p.C = part_embed;
    DZ_TRY(launch_pgemm("iqn_embed_wgrad", kb, l->side.fork(stream, stream)));
    fb.f[fb.n++] = FinishTN{p.C, p.splits, p.split_stride, c.latent_dim, d.feat, G + o.embed_w, nullptr, G + o.embed_b, nullptr, nullptr, nullptr};
  } else {
    DZ_TRY(launch_iqn_hadamard_bwd(false, l->dhi, l->E0, l->act3[0], l->dact3, nullptr, nullptr, 0, B, N, d.feat, stream));
    {  // embed wgrad: [latent, feat] = cos^T * dE
      GemmProblem p = zero_problem();
      p.a_mode = A_PLAIN; p.A = l->cosf[0]; p.lda = c.latent_dim; p.M = M; p.K = c.latent_dim;
      p.B = l->dhi; p.N = d.feat; p.ldb = d.feat; p.ldc = d.feat;
      p.Cb = G + o.embed_b;
      int splits = (int)std::min<int64_t>(16, ceil_div(M, 64));
      p.splits = splits; p.split_stride = (long long)(c.latent_dim + 1) * d.feat; p.C = part_embed;
      gb.p[0] = p;
      DZ_TRY(run_tn("iqn_embed_wgrad", gb, l->side.fork(stream, stream)));
      fb.f[fb.n++] = FinishTN{p.C, splits, p.split_stride, c.latent_dim, d.feat, G + o.embed_w, nullptr, p.Cb, nullptr, nullptr, nullptr};
    }
  }
  long long mx = 0;
  for (int q = 0; q < fb.n; ++q) mx = std::max<long long>(mx, (long long)(fb.f[q].K + 1) * fb.f[q].N);
  dim3 grid((unsigned)std::min<long long>(ceil_div(mx, 256), kNumSMs * 8), fb.n);
  DZ_LAUNCH(finish_tn_kernel, grid, 256, 0, l->side.tail(stream), fb);
  return DZ_OK;
}

// fqf: fraction_forward_kernel over E examples of `napp` applications (grid E x napp), reading the fraction layer of
// `params` (the online blob, or a frozen actor's snapshot).
int launch_fraction_forward(const dz_learner* l, FracArgs f, const float* params, int E, int napp, void* stream) {
  f.W = params + l->po.frac_w; f.bias = params + l->po.frac_b;
  f.N = l->cfg.num_fractions; f.D = l->d.feat;
  DZ_LAUNCH(fraction_forward_kernel, dim3((unsigned)E, (unsigned)napp), 256, 0, stream, f);
  return DZ_OK;
}

// fqf's acting forward on set 1 of `nb` (the torso has run): the fraction layer of `params` on act3, then one N-row
// IQN pass at tau_hat; the interval weights land in `w` for the q-values.
int fqf_act_heads(dz_learner* l, const NetBufs& nb, const float* params, int E, float* hat, float* w, void* stream) {
  FracArgs f;
  memset(&f, 0, sizeof(f));
  f.feat[0] = nb.act3[1]; f.tau_hat[0] = hat; f.w[0] = w;
  DZ_TRY(launch_fraction_forward(l, f, params, E, 1, stream));
  Pass pass{params, 1, 1, 0};
  const float* taus[1] = {hat};
  return forward_heads_iqn(l, nb, &pass, 1, E, taus, false, stream, true);
}

// fqf: the fraction layer's gradient, dW_f = act3(s_tm1)^T dlogits ([feat][N], rank B) and db_f = sum_b dlogits, on the
// fp32 TN GEMM on the side stream (the features are stop-gradient: nothing flows back into the torso).
int backward_fraction(dz_learner* l, void* stream) {
  const Dims& d = l->d;
  const ParamOffsets& o = l->po;
  const int N = l->cfg.num_fractions;
  float* G = l->buf.d_grads;
  GemmBatch gb;
  gb.n = 1;
  GemmProblem p = zero_problem();
  p.a_mode = A_PLAIN; p.A = l->act3[0]; p.lda = d.feat; p.M = l->B; p.K = d.feat;
  p.B = l->fq_dlogits; p.N = N; p.ldb = N; p.ldc = N;
  p.C = G + o.frac_w; p.Cb = G + o.frac_b;
  gb.p[0] = p;
  return run_tn("fqf_fraction_wgrad", gb, l->side.fork(stream, stream));
}

// Split global norm (tensor-core path, every agent but IQN): the sum of squares of everything behind the conv tensors is taken
// on the second side stream as soon as the last FC / head weight gradient is written (norm_fc_range), the conv tensors'
// partials come from the per-layer weight-gradient finish kernels, and the optimizer (or norm_finalize_kernel) combines them.
bool split_norm_active(const dz_learner* l) { return l->um != nullptr && !uses_iqn_net(l->cfg.kind); }

int norm_fc_range(dz_learner* l, bool apply, void* stream) {
  const long long begin = l->po.fc_begin;
  const long long n = l->lay.total - begin;
  DZ_LAUNCH(grad_norm_kernel, kNormBlocks, 256, 0, stream, l->buf.d_grads + begin, n, l->scalars + 8, l->ticket, l->scalars + 1,
            apply ? l->buf.d_counters : l->buf.d_counters + 3, (float*)nullptr, 1);
  return DZ_OK;
}

int run_optimizer(dz_learner* l, float* user_norm, bool apply, void* stream) {
  const dz_learner_config& c = l->cfg;
  long long n = l->lay.total;
  // fqf: the norm, the clip and the configured optimizer cover [0, frac_w); the fraction tail gets its own launch below
  const bool frac = proposes_fractions(c.kind);
  const long long n_main = frac ? l->po.frac_w : n;
  float* norm = l->scalars;
  const bool split = split_norm_active(l);
  const float* parts = split ? l->norm_parts : nullptr;
  const int nparts = split ? um_norm_slots(l->um) : 0;
  if (!split) {
    DZ_LAUNCH(grad_norm_kernel, kNormBlocks, 256, 0, stream, l->buf.d_grads, n_main, l->scalars + 8, l->ticket, norm,
              apply ? l->buf.d_counters : l->buf.d_counters + 3, user_norm, 0);
  } else if (!apply) {
    DZ_LAUNCH(norm_finalize_kernel, 1, 256, 0, stream, parts, nparts, l->scalars + 1, norm, user_norm);
  }
  if (!apply) return DZ_OK;
  OptArgs o{c.optimizer, c.learning_rate, c.opt_eps, c.rms_decay, c.adam_b1, c.adam_b2, c.max_global_grad_norm,
            l->buf.d_online, l->buf.d_grads, l->buf.d_opt_state, l->buf.d_opt_state + n, n_main, norm, l->buf.d_counters,
            parts, nparts, l->scalars + 1, norm, user_norm};
  o.stages = kOptRingStages;
  const OptKernel kernel = optimizer_kernel_for(c.optimizer);
  const OptKernel frac_kernel = optimizer_kernel_for(DZ_RMSPROP_CENTERED);
  if (!l->opt_smem_set) {
    DZ_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kOptSmem));
    if (frac) DZ_CUDA_OK(cudaFuncSetAttribute(frac_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kOptSmem));
    l->opt_smem_set = true;
  }
  auto grid_of = [](long long count) {
    const long long nchunks = ((count >> 2) + kOptChunk - 1) / kOptChunk;
    return (unsigned)std::max<long long>(1, std::min<long long>((long long)kNumSMs * kOptBlocksPerSM, nchunks));
  };
  DZ_LAUNCH_NAMED("optimizer_kernel", kernel, grid_of(o.n), kOptThreads, kOptSmem, stream, o);
  if (frac) {   // centred RMSProp over the fraction layer, without a clip, on the same moment buffers at the same offsets
    const long long fb = l->po.frac_w;
    OptArgs f{DZ_RMSPROP_CENTERED, c.fraction_learning_rate, c.fraction_opt_eps, c.fraction_rms_decay, c.adam_b1, c.adam_b2,
              0.f, l->buf.d_online + fb, l->buf.d_grads + fb, l->buf.d_opt_state + fb, l->buf.d_opt_state + n + fb, n - fb,
              norm, l->buf.d_counters, nullptr, 0, nullptr, nullptr, nullptr};
    f.stages = kOptRingStages;
    DZ_LAUNCH_NAMED("fqf_fraction_optimizer", frac_kernel, grid_of(f.n), kOptThreads, kOptSmem, stream, f);
  }
  return DZ_OK;
}

// The loss section of a learner step: the agent kind's loss kernel on `stream`, then loss_mean_kernel (the scalar loss,
// and the running max priority when max_seen is given and the learner writes priorities).  L carries the buffers: head
// outputs, batch, outputs and loss_terms; every field that follows from the configuration (sizes, vmax, bound, kappa,
// whether priorities are written: writes_priorities) is set here.  With `side`, loss_mean_kernel runs on the side stream forked after the loss kernel and
// *mean_stream receives it; without, everything runs on `stream`.  dz_test_loss and dz_test_loss_fqf run this same
// function.
// cql_alpha > 0 (DESIGN.md §20) selects each kernel's cql variant, which writes R_b to `regularizer` when it is given;
// the launch count is the same at every alpha.
int launch_loss(const dz_learner_config& c, LossArgs& L, int B, void* stream, SideStream* side, float* d_loss, float* max_seen,
                void** mean_stream, const FqfLossArgs* fqf = nullptr, float* regularizer = nullptr) {
  L.kind = c.kind; L.B = B; L.A = c.num_actions; L.atoms = c.num_atoms;
  L.vmax = c.vmax; L.bound = c.grad_error_bound; L.kappa = c.huber_param;
  if (!writes_priorities(c)) L.priorities = nullptr;
  const bool cql = c.cql_alpha > 0.f;
  const CqlArgs cq{c.cql_alpha, regularizer};
#define DZ_LAUNCH_LOSS(name, kernel, grid, block, smem, ...)                                   \
  do {                                                                                         \
    if (cql) DZ_LAUNCH_NAMED(name, kernel<true>, grid, block, smem, stream, __VA_ARGS__, cq);  \
    else DZ_LAUNCH_NAMED(name, kernel<false>, grid, block, smem, stream, __VA_ARGS__, cq);     \
  } while (0)
  if (c.kind == DZ_DQN || c.kind == DZ_DOUBLE_Q || c.kind == DZ_PRIORITIZED) {
    DZ_LAUNCH_LOSS("loss_q_kernel", loss_q_kernel, B, 64, 0, L);
  } else if (c.kind == DZ_MUNCHAUSEN) {
    DZ_LAUNCH_LOSS("loss_munchausen_kernel", loss_munchausen_kernel, (B + 3) / 4, 128, 0, L, c.munchausen_alpha,
                   c.entropy_temperature, c.log_policy_clip);
  } else if (c.kind == DZ_C51 || c.kind == DZ_RAINBOW) {
    // More than the default 48 KB of dynamic shared memory at large num_actions x num_atoms; the attribute is per
    // device, so it is set for the current one.
    const size_t smem = categorical_loss_smem(c);
    if (smem > 48 * 1024)
      DZ_CUDA_OK(cudaFuncSetAttribute(cql ? loss_categorical_staged_kernel<true> : loss_categorical_staged_kernel<false>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    DZ_LAUNCH_LOSS("loss_categorical_kernel", loss_categorical_staged_kernel, B, 128, smem, L);
  } else if (proposes_fractions(c.kind)) {
    if (!fqf) return fail(DZ_EINVAL, "fqf's loss needs the fraction buffers of a learner step");
    L.N = c.num_fractions; L.Ksel = c.num_fractions; L.Nt = c.num_fractions;
    DZ_LAUNCH_LOSS("loss_fqf_kernel", loss_fqf_kernel, B, 256, fqf_loss_smem(c), L, *fqf);
  } else if (c.kind == DZ_MUNCHAUSEN_IQN) {
    L.N = c.tau_samples_s_tm1; L.Ksel = c.tau_samples_policy; L.Nt = c.tau_samples_s_t;
    DZ_LAUNCH_LOSS("loss_munchausen_iqn_kernel", loss_munchausen_iqn_kernel, B, 256, munchausen_iqn_loss_smem(c), L,
                   c.munchausen_alpha, c.entropy_temperature, c.log_policy_clip);
  } else {
    if (c.kind == DZ_QRDQN) { L.N = c.num_quantiles; L.Ksel = c.num_quantiles; L.Nt = c.num_quantiles; }
    else { L.N = c.tau_samples_s_tm1; L.Ksel = c.tau_samples_policy; L.Nt = c.tau_samples_s_t; }
    size_t smem = (32 + c.num_actions + L.Nt + 2 * L.N + (cql ? 2 * c.num_actions + 1 : 0)) * sizeof(float);
    DZ_LAUNCH_LOSS("loss_quantile_kernel", loss_quantile_kernel, B, 256, smem, L);
  }
#undef DZ_LAUNCH_LOSS
  void* ms = side ? side->fork(stream, stream) : stream;
  DZ_LAUNCH(loss_mean_kernel, 1, 32, 0, ms, L.loss_terms, B, d_loss, max_seen, L.priorities);
  if (mean_stream) *mean_stream = ms;
  return DZ_OK;
}

// The acting tail of a head pass over E observations: q-values [E][A] (q_values_kernel) and, when `actions` is given,
// the epsilon-greedy choice (act_select_kernel).  out: the head outputs of the pass (rainbow: the advantage stream),
// val: rainbow's value stream.  The acting body (the learner's and the actor's), dz_test_q_values and
// dz_test_q_values_fqf run this function.
// fqf: `frac_w` holds the interval weights [E][N] of the pass's proposals (q_values_fqf_kernel).
int launch_q_values(const dz_learner_config& c, int E, const float* out, const float* val, const float* explore, float epsilon,
                    float* q, int32_t* actions, void* stream, const float* frac_w = nullptr) {
  if (proposes_fractions(c.kind)) {
    if (!frac_w) return fail(DZ_EINVAL, "fqf's q-values need the interval weights of the acting pass's proposals");
    DZ_LAUNCH(q_values_fqf_kernel, (unsigned)E, 64, 0, stream, c.num_actions, c.num_fractions, out, frac_w, q);
  } else {
    const int nq = uses_iqn_net(c.kind) ? c.tau_samples_policy : c.num_quantiles;
    const size_t smem = (32 + c.num_atoms + 8) * sizeof(float);
    DZ_LAUNCH(q_values_kernel, (unsigned)E, 128, smem, stream, net_kind(c.kind), c.num_actions, c.num_atoms, nq, c.vmax, out,
              out, val, q);
  }
  if (actions)
    DZ_LAUNCH(act_select_kernel, (unsigned)ceil_div(E, 128), 128, 0, stream, (const float*)q, c.num_actions, E, explore, epsilon,
              actions);
  return DZ_OK;
}

// What one act reads and writes.  The learner's acting fills it with its own fp32 buffers (split-K up to 32 rows), its
// row table and fqf buffers, and no plan; an actor with buffers sized for its streams and, where the geometry allows,
// its forward-only tensor-core plan.
struct ActTarget {
  dz_learner* l;              // configuration, layout, offsets, dims and split counts (a frozen actor's: shape only)
  const float* params;        // the online blob or a frozen snapshot
  NetBufs nb;                 // activation set / head pass 1
  const uint8_t** rows;       // [E] observation row table
  UmNet* um;                  // forward-only tensor-core plan (nullptr: fp32-FMA torso)
  bool pack;                  // pack the plan's weight images on every act (a live actor; frozen: packed by load_params)
  float* noise;               // rainbow on the plan: the copy of the caller's shared apply that noisy1 reads
  float *frac_hat, *frac_w;   // fqf: the acting pass's tau_hat and interval weights, [E][N] each
};

// The acting body of dz_learner_act_batch and dz_actor_act: row table, torso, heads by kind, q-values and, when
// d_actions is given, the epsilon-greedy choice.
int act(const ActTarget& t, int E, const uint8_t* d_obs, const float* d_taus, const float* d_noise, int64_t noise_ld,
        const float* d_explore, float epsilon, float* d_q_out, int32_t* d_actions, void* stream) {
  dz_learner* l = t.l;
  const dz_learner_config& c = l->cfg;
  const bool rb = noisy_net(c);
  if (!d_obs || !d_q_out) return fail(DZ_EINVAL, "act: null buffer");
  if (draws_taus(c.kind) && !d_taus) return fail(DZ_EINVAL, "iqn acting needs taus[E][tau_samples_policy]");
  if (rb && !d_noise) return fail(DZ_EINVAL, "acting a noisy network needs noise");
  const int64_t stride = rb ? noise_layout(c, l->d).stride : 0;
  if (noise_ld != 0 && (!rb || noise_ld != stride))
    return fail(DZ_EINVAL, "act: noise_ld must be 0 (one shared apply) or the noise stride (noisy layers, one apply per stream)");
  const float* on = t.params;
  const long long obs_bytes = (long long)l->d.H * l->d.W * l->d.C;
  DZ_LAUNCH(make_row_table_kernel, (unsigned)ceil_div(E, 64), 64, 0, stream, d_obs, obs_bytes, E, t.rows);
  const bool fc_done = t.um && !uses_iqn_net(c.kind) && noise_ld == 0;
  if (t.um) {
    const uint8_t* const* rows[3] = {t.rows, nullptr, nullptr};
    if (t.pack) DZ_TRY(um_pack_weights(t.um, stream));
    DZ_TRY(um_forward_torso(t.um, rows, stream));
    if (fc_done) {
      if (rb) DZ_CUDA_OK(cudaMemcpyAsync(t.noise, d_noise, stride * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
      DZ_TRY(um_forward_fc(t.um, t.noise, stream));
    }
  } else {
    TorsoJob job{on, t.rows, 1};   // activation set 1, so a pending backward's set-0 buffers stay intact
    DZ_TRY(forward_torso(l, t.nb, &job, 1, E, stream));
  }
  Pass pass{on, 1, 1, 0};
  if (proposes_fractions(c.kind)) {
    DZ_TRY(fqf_act_heads(l, t.nb, on, E, t.frac_hat, t.frac_w, stream));
  } else if (uses_iqn_net(c.kind)) {
    const float* taus[1] = {d_taus};
    DZ_TRY(forward_heads_iqn(l, t.nb, &pass, 1, E, taus, false, stream));
  } else {
    DZ_TRY(forward_heads_fc(l, t.nb, &pass, 1, E, d_noise, stream, fc_done, noise_ld));
  }
  return launch_q_values(c, E, t.nb.out[1], t.nb.outv[1], d_explore, epsilon, d_q_out, d_actions, stream, t.frac_w);
}

// One draw of acting randomness: n floats from the generator of dz_learner_generate_randomness (Philox keyed by element
// index, counter counters[1] and the stream id of its taus or of its noise), then one counter step.
int launch_acting_draw(float* d_out, long long n, bool taus, uint64_t seed, int64_t* counters, void* stream) {
  DZ_LAUNCH(randomness_kernel, (unsigned)ceil_div(ceil_div(n, 4), 256), 256, 0, stream, d_out, n, seed, counters, taus ? 0 : 1,
            taus ? 1u : 2u);
  DZ_LAUNCH(bump_counter_kernel, 1, 1, 0, stream, counters, 1);
  return DZ_OK;
}

// random_shift_kernel over B examples: d_out [B][2][stride]; rows_tm1 / rows_t (or NULL) are pointed at the results.
int launch_random_shift(const uint8_t* const* src_tm1, const uint8_t* const* src_t, const int32_t* shifts, int B, int H, int W,
                        int C, int pad, uint8_t* out, long long stride, const uint8_t** rows_tm1, const uint8_t** rows_t,
                        void* stream) {
  const ShiftArgs a{{src_tm1, src_t}, shifts, out, stride, {rows_tm1, rows_t}, H, W, C, pad};
  DZ_LAUNCH(random_shift_kernel, dim3(2, (unsigned)B), kShiftThreads, 0, stream, a);
  return DZ_OK;
}

// The step's shifted observations (DESIGN.md §18): the batch's row tables, whatever the sampler or the caller pointed
// them at (replay rows, the frame-deduplicated reconstruction, dense arrays), into l->shift_obs and l->rows_shift.
int launch_learner_shift(dz_learner* l, const dz_batch* batch, void* stream) {
  const Dims& d = l->d;
  const long long obs = (long long)d.H * d.W * d.C;
  return launch_random_shift(batch->d_s_tm1_rows, batch->d_s_t_rows, batch->d_shifts, l->B, d.H, d.W, d.C,
                             l->cfg.random_shift_pad, l->shift_obs, obs, l->rows_shift[0], l->rows_shift[1], stream);
}

struct WriteBack { const dz_replay_view* view; const int64_t* indices; const float* priorities; double alpha; };

int update_impl(dz_learner* l, const dz_batch* batch, const dz_update_outputs* out, int apply_update, float* max_seen,
                const WriteBack* wb, void* stream, bool weights_packed = false) {
  const dz_learner_config& c = l->cfg;
  const int B = l->B;
  const float* on = l->buf.d_online;
  const float* tg = l->buf.d_target;
  const bool online_st = online_applies_to_s_t(c.kind);
  if (noisy_net(c) && !batch->d_noise) return fail(DZ_EINVAL, "a noisy network's update needs d_noise");
  if (draws_taus(c.kind) && !batch->d_taus) return fail(DZ_EINVAL, "iqn update needs d_taus");
  if (!out || !out->d_loss || !out->d_per_example) return fail(DZ_EINVAL, "update outputs d_loss and d_per_example are required");
  const bool shift = c.random_shift_pad > 0;
  if (shift && !batch->d_shifts) return fail(DZ_EINVAL, "an update with random_shift_pad > 0 needs d_shifts");
  if (!(weights_packed && l->um != nullptr)) DZ_TRY(l->side.join(stream));   // pending side-stream work (asynchronous randomness)

  // ---- forward: every network.apply of loss_fn in grouped launches.  With augmentation every pass over s_tm1 reads
  // the one shifted s_tm1 and every pass over s_t the one shifted s_t (DESIGN.md §18).
  const uint8_t* const* s_tm1 = shift ? l->rows_shift[0] : batch->d_s_tm1_rows;
  const uint8_t* const* s_t = shift ? l->rows_shift[1] : batch->d_s_t_rows;
  TorsoJob jobs[3];
  int nj = 0;
  const bool target_stm1 = is_munchausen(c.kind);   // the target network also applies to s_tm1 (the log-policy bonus)
  const bool iqn = uses_iqn_net(c.kind);
  jobs[nj++] = TorsoJob{on, s_tm1, 0};
  if (online_st) jobs[nj++] = TorsoJob{on, s_t, 1};
  if (target_stm1) jobs[nj++] = TorsoJob{tg, s_tm1, 1};
  jobs[nj++] = TorsoJob{tg, s_t, 2};
  const bool um = l->um != nullptr;
  if (um) {
    if (nj != l->um_npass) return fail(DZ_EINVAL, "tensor-core path: pass count mismatch");
    const uint8_t* const* rows[3] = {nullptr, nullptr, nullptr};
    for (int i = 0; i < nj; ++i) rows[i] = jobs[i].rows;
    if (weights_packed) DZ_TRY(l->side.join(stream));   // packed on the side stream, concurrently with the sampler
    else DZ_TRY(um_pack_weights(l->um, stream));
    if (shift) DZ_TRY(launch_learner_shift(l, batch, stream));   // after the join: the shifts may be drawn beside the sampler
    DZ_TRY(um_forward_torso(l->um, rows, stream));
    DZ_TRY(l->side.join(stream));
    if (!iqn) DZ_TRY(um_forward_fc(l->um, batch->d_noise, stream));
  } else {
    if (shift) DZ_TRY(launch_learner_shift(l, batch, stream));
    DZ_TRY(forward_torso(l, learner_bufs(l), jobs, nj, B, stream));
  }

  const bool fqf = proposes_fractions(c.kind);
  if (fqf) {
    // fqf: the fraction layer on online(s_tm1)'s and target(s_t)'s features, then online(s_tm1, tau_hat) |
    // online(s_tm1, tau_1..tau_N) (no gradient) | target(s_t, [tau_hat' | tau_hat])   (DESIGN.md §15)
    const long long n = (long long)B * c.num_fractions;
    FracArgs f;
    memset(&f, 0, sizeof(f));
    f.feat[0] = l->act3[0]; f.feat[1] = l->act3[2];
    for (int a = 0; a < 2; ++a) {
      f.tau[a] = l->fq_tau + a * (n + B); f.tau_hat[a] = l->fq_hat + a * n; f.w[a] = l->fq_w + a * n; f.q[a] = l->fq_q + a * n;
    }
    f.pass1 = l->fq_pass1; f.pass2 = l->fq_pass2;
    DZ_TRY(launch_fraction_forward(l, f, on, B, 2, stream));
    Pass passes[3] = {{on, 0, 0, 0}, {on, 0, 1, 0}, {tg, 2, 2, 0}};
    const float* taus[3] = {l->fq_hat, l->fq_pass1, l->fq_pass2};
    DZ_TRY(forward_heads_iqn(l, learner_bufs(l), passes, 3, B, taus, true, stream));
  } else if (iqn) {
    // iqn: online(s_tm1, tau_tm1) | target(s_t, tau_selector) | target(s_t, tau_t)   (iqn/agent.py:192-203)
    // munchausen_iqn: online(s_tm1, tau_tm1) | target(s_tm1, tau_policy) | target(s_t, tau_t), three torso sets
    Pass passes[3] = {{on, 0, 0, 0}, {tg, target_stm1 ? 1 : 2, 1, 0}, {tg, 2, 2, 0}};
    const float* t0 = batch->d_taus;
    const float* t1 = t0 + (long long)B * c.tau_samples_s_tm1;
    const float* t2 = t1 + (long long)B * c.tau_samples_policy;
    const float* taus[3] = {t0, t1, t2};
    DZ_TRY(forward_heads_iqn(l, learner_bufs(l), passes, 3, B, taus, true, stream));
  } else {
    // noise slot = head pass (rainbow, noisy networks, DESIGN.md §17): online(s_tm1) | the middle pass | target(s_t)
    Pass passes[3];
    int np = 0;
    passes[np++] = Pass{on, 0, 0, 0};
    if (online_st) passes[np++] = Pass{on, 1, 1, 1};
    if (target_stm1) passes[np++] = Pass{tg, 1, 1, 1};
    passes[np++] = Pass{tg, 2, 2, 2};
    DZ_TRY(forward_heads_fc(l, learner_bufs(l), passes, np, B, batch->d_noise, stream, um, 0, true));
  }

  // ---- loss + gradient wrt the pass-0 head outputs
  LossArgs L;
  memset(&L, 0, sizeof(L));
  L.out0 = l->out[0]; L.out1 = l->out[1]; L.out2 = l->out[2];
  L.adv0 = l->out[0]; L.val0 = l->outv[0]; L.adv1 = l->out[1]; L.val1 = l->outv[1]; L.adv2 = l->out[2]; L.val2 = l->outv[2];
  L.a = batch->d_a_tm1; L.r = batch->d_r_t; L.disc = batch->d_discount_t; L.w = batch->d_weights;
  L.taus0 = fqf ? l->fq_hat : batch->d_taus;
  L.dout = l->dout; L.dadv = l->dout; L.dval = l->doutv;
  L.per_example = out->d_per_example; L.loss_terms = l->loss_terms; L.priorities = out->d_priorities;
  const FqfLossArgs fl{l->fq_w + (fqf ? (long long)B * c.num_fractions : 0), l->fq_q, l->fq_dlogits};
  {   // the scalar loss / running max priority and replay.update_priorities(ids, priorities) (rainbow/agent.py:198) are
      // independent of the backward pass: both leave the critical path for the side stream
    void* ls = stream;
    DZ_TRY(launch_loss(c, L, B, stream, &l->side, out->d_loss, max_seen, &ls, fqf ? &fl : nullptr, out->d_regularizer));
    if (wb) DZ_TRY(launch_update_priorities(wb->view, wb->indices, wb->priorities, B, wb->alpha, wb->view->capacity, ls));
  }

  // ---- backward through online(s_tm1)
  if (iqn) DZ_TRY(backward_iqn(l, stream));
  else DZ_TRY(backward_fc(l, batch->d_noise, stream));
  if (fqf) DZ_TRY(backward_fraction(l, stream));
  if (split_norm_active(l)) {   // every gradient behind the conv tensors is final once the side stream's FC / head wgrads are done
    DZ_TRY(norm_fc_range(l, apply_update != 0, l->side.tail(stream)));
  }
  DZ_TRY(backward_torso(l, s_tm1, stream));

  // ---- clip_by_global_norm + adam / rmsprop + apply_updates
  DZ_TRY(l->side2.join(stream));
  DZ_TRY(l->side.join(stream));
  DZ_TRY(run_optimizer(l, out->d_grad_norm, apply_update != 0, stream));
  return DZ_OK;
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------

extern "C" {

int dz_learner_plan_query(const dz_learner_config* cfg, dz_learner_plan* out) {
  DZ_TRY(validate(*cfg));
  dz_learner tmp;
  out->workspace_bytes = init_shape_learner(&tmp, *cfg);
  out->param_count = tmp.lay.total;
  out->num_tensors = (int32_t)tmp.lay.t.size();
  out->opt_state_floats = 2 * tmp.lay.total;
  out->noise_floats = noisy_net(*cfg) ? 3 * noise_layout(*cfg, tmp.d).stride : 0;
  out->tau_floats = draws_taus(cfg->kind)
                        ? (int64_t)cfg->batch * (cfg->tau_samples_s_tm1 + cfg->tau_samples_policy + cfg->tau_samples_s_t)
                        : 0;
  return DZ_OK;
}

int dz_learner_tensor_info(const dz_learner_config* cfg, int32_t i, char* name64, int64_t* shape4, int32_t* ndim, int64_t* offset) {
  DZ_TRY(validate(*cfg));
  Layout L = make_layout(*cfg);
  if (i < 0 || i >= (int)L.t.size()) return fail(DZ_ERANGE, "tensor index out of range");
  const TensorInfo& t = L.t[i];
  snprintf(name64, 64, "%s", t.name.c_str());
  for (int k = 0; k < 4; ++k) shape4[k] = t.shape[k];
  *ndim = t.ndim;
  *offset = t.offset;
  return DZ_OK;
}

int dz_learner_create(const dz_learner_config* cfg, const dz_learner_buffers* buf, dz_learner** out) {
  DZ_TRY(validate(*cfg));
  if (!buf->d_online || !buf->d_target || !buf->d_grads || !buf->d_opt_state || !buf->d_workspace || !buf->d_counters)
    return fail(DZ_EINVAL, "all learner buffers are required");
  dz_learner* l = new dz_learner();
  init_shape_learner(l, *cfg);
  l->buf = *buf;
  carve(l, static_cast<char*>(buf->d_workspace));
  if (l->um_ws) {
    UmNetDesc ud = make_um_desc(l);
    const int rc = um_net_create(ud, l->um_ws, &l->um);
    if (rc != DZ_OK) { delete l; return rc; }
    l->um_npass = ud.npass;
    const int um_set[3] = {0, ud.npass == 3 ? 1 : 2, 2};   // torso activation set of each tensor-core pass
    for (int i = 0; i < ud.npass; ++i) {   // the fp32 views the remaining FMA kernels, the losses and the tests read
      const int set = um_set[i];
      l->act1[set] = um_act_f32(l->um, 1, i); l->act2[set] = um_act_f32(l->um, 2, i); l->act3[set] = um_act_f32(l->um, 3, i);
      if (ud.use_fc)
        for (int s = 0; s < ud.nstream; ++s) l->h1[set][s] = um_h1_f32(l->um, i, s);
    }
    if (ud.use_fc)
      for (int s = 0; s < ud.nstream; ++s) l->dh1[s] = um_dh1_f32(l->um, s);
    l->dact3 = um_dact_f32(l->um, 3); l->dact2 = um_dact_f32(l->um, 2); l->dact1 = um_dact_f32(l->um, 1);
  }
  cudaError_t se = l->side.create();
  if (se == cudaSuccess) se = l->side2.create();
  if (se == cudaSuccess) se = l->side3.create();
  if (se != cudaSuccess) { dz_learner_destroy(l); return fail(DZ_ECUDA, "side streams: %s", cudaGetErrorString(se)); }
  if (l->pk_on) {
    // fused epilogues only write the valid region of these images: zero the padding once, and set the constant
    // row of ones (bias-gradient row) of the transposed activation image
    for (int p = 0; p < 3; ++p) {
      cudaMemset(l->pk_act[p].hi, 0, pk_image_floats(l->pk_act[p].rows_pad, l->pk_act[p].red_pad) * sizeof(float));
      cudaMemset(l->pk_act[p].lo, 0, pk_image_floats(l->pk_act[p].rows_pad, l->pk_act[p].red_pad) * sizeof(float));
    }
    cudaMemset(l->pk_actT.hi, 0, pk_image_floats(l->pk_actT.rows_pad, l->pk_actT.red_pad) * sizeof(float));
    cudaMemset(l->pk_actT.lo, 0, pk_image_floats(l->pk_actT.rows_pad, l->pk_actT.red_pad) * sizeof(float));
    if (l->pk_embed_bwd) {
      cudaMemset(l->pk_dET.hi, 0, pk_image_floats(l->pk_dET.rows_pad, l->pk_dET.red_pad) * sizeof(float));
      cudaMemset(l->pk_dET.lo, 0, pk_image_floats(l->pk_dET.rows_pad, l->pk_dET.red_pad) * sizeof(float));
    }
    int rc = pk_set_ones_row(l->pk_actT.hi, l->pk_actT.rows_pad, l->d.feat, l->B * l->n_head[0], nullptr);
    if (rc != DZ_OK || cudaDeviceSynchronize() != cudaSuccess) { delete l; return rc != DZ_OK ? rc : fail(DZ_ECUDA, "packed image init"); }
  }
  cudaError_t e = cudaMemset(l->ticket, 0, 16);
  if (e != cudaSuccess) { delete l; return fail(DZ_ECUDA, "cudaMemset: %s", cudaGetErrorString(e)); }
  *out = l;
  return DZ_OK;
}

void dz_learner_destroy(dz_learner* l) {
  if (!l) return;
  um_net_destroy(l->um);
  l->side.destroy();
  l->side2.destroy();
  l->side3.destroy();
  if (l->recon) cudaFree(l->recon);
  delete l;
}

int dz_learner_update(dz_learner* l, const dz_batch* batch, const dz_update_outputs* out, int32_t apply_update, void* stream) {
  return update_impl(l, batch, out, apply_update, nullptr, nullptr, stream);
}

int dz_learner_learn(dz_learner* l, const dz_replay_view* replay, int32_t prioritized, const dz_learn_io* io, void* stream) {
  const int B = l->B;
  if (prioritized && !writes_priorities(l->cfg))
    return fail(DZ_EINVAL, "prioritized learn needs a learner that writes priorities (prioritized, rainbow, or "
                           "dz_learner_config.prioritized = 1)");
  BatchExtras ex{l->rows_sample[0], l->rows_sample[1], l->s_a, l->s_r, l->s_d, prioritized ? l->s_w : nullptr, 1};
  if (replay->obs_bytes != (int64_t)l->d.H * l->d.W * l->d.C) return fail(DZ_EINVAL, "replay observation size does not match the network");
  if (replay->d_planes) {
    const int64_t need = (int64_t)B * 2 * replay->obs_stride;
    if (need > l->recon_bytes) {
      cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
      DZ_CUDA_OK(cudaStreamIsCapturing((cudaStream_t)stream, &cs));
      if (cs != cudaStreamCaptureStatusNone)
        return fail(DZ_EINVAL, "the first dz_learner_learn on a frame-deduplicated replay must run eagerly, not in a capture");
      if (l->recon) DZ_CUDA_OK(cudaFree(l->recon));
      l->recon = nullptr;
      l->recon_bytes = 0;
      DZ_CUDA_OK(cudaMalloc(&l->recon, need));
      l->recon_bytes = need;
    }
    ex.recon = l->recon;
  }
  // conv weight images do not depend on the sampled batch: pack them on the side stream while the sampler runs
  const bool pack_aside = l->um != nullptr;
  if (pack_aside) {
    void* ws = l->side.fork(stream, stream);
    DZ_TRY(um_pack_weights(l->um, ws));
  }
  DZ_TRY(launch_sample(replay, prioritized, &io->sample_in, &io->sample_out, B, ex, stream));
  if (replay->d_planes)
    DZ_TRY(launch_frame_reconstruct(replay, io->sample_out.d_slots, B, l->recon, l->recon + replay->obs_stride,
                                    2 * replay->obs_stride, stream));
  dz_batch batch;
  batch.d_s_tm1_rows = l->rows_sample[0];
  batch.d_s_t_rows = l->rows_sample[1];
  batch.d_a_tm1 = l->s_a; batch.d_r_t = l->s_r; batch.d_discount_t = l->s_d;
  batch.d_weights = prioritized ? l->s_w : nullptr;
  batch.d_taus = io->d_taus; batch.d_noise = io->d_noise;
  batch.d_shifts = l->cfg.random_shift_pad ? io->d_shifts : nullptr;   // the field is not read with the pad at 0
  WriteBack wb{replay, io->sample_out.d_indices, io->update_out.d_priorities, io->priority_exponent};
  if (prioritized && !io->update_out.d_priorities) return fail(DZ_EINVAL, "prioritized learn needs update_out.d_priorities");
  DZ_TRY(update_impl(l, &batch, &io->update_out, 1, io->d_max_seen_priority, prioritized ? &wb : nullptr, stream, pack_aside));
  return DZ_OK;
}

// Same as dz_learner_generate_randomness, but enqueued on the learner's side stream (when it has one): the draws do not
// depend on the sampled batch, so they run beside the sampler instead of in front of it.  Ordered after everything already
// enqueued on `stream` and before the next dz_learner_learn / dz_learner_update / dz_learner_act_batch on `stream`; any
// other consumer of the buffers must synchronise the device first.
int dz_learner_generate_randomness_async(dz_learner* l, uint64_t seed, float* d_taus, float* d_noise, void* stream) {
  return dz_learner_generate_randomness(l, seed, d_taus, d_noise, l->side.fork(stream, stream));
}

// The shifts of the next update at the current counter; the dz_learner_generate_randomness enqueued after it makes the
// step's one counter step.
int dz_learner_generate_shifts(dz_learner* l, uint64_t seed, int32_t* d_shifts, void* stream) {
  if (l->cfg.random_shift_pad == 0) return fail(DZ_EINVAL, "generate_shifts: the learner's random_shift_pad is 0");
  if (!d_shifts) return fail(DZ_EINVAL, "generate_shifts: null buffer");
  DZ_LAUNCH(shift_draw_kernel, (unsigned)ceil_div(l->B, 128), 128, 0, stream, d_shifts, l->B, l->cfg.random_shift_pad, seed,
            l->buf.d_counters);
  return DZ_OK;
}

int dz_learner_generate_randomness(dz_learner* l, uint64_t seed, float* d_taus, float* d_noise, void* stream) {
  const dz_learner_config& c = l->cfg;
  if (draws_taus(c.kind) && d_taus) {
    long long n = (long long)c.batch * (c.tau_samples_s_tm1 + c.tau_samples_policy + c.tau_samples_s_t);
    DZ_LAUNCH(randomness_kernel, (unsigned)ceil_div(ceil_div(n, 4), 256), 256, 0, stream, d_taus, n, seed, l->buf.d_counters, 0, 1u);
  }
  if (noisy_net(c) && d_noise) {
    long long n = 3 * noise_layout(c, l->d).stride;
    DZ_LAUNCH(randomness_kernel, (unsigned)ceil_div(ceil_div(n, 4), 256), 256, 0, stream, d_noise, n, seed, l->buf.d_counters, 1, 2u);
  }
  DZ_LAUNCH(bump_counter_kernel, 1, 1, 0, stream, l->buf.d_counters, 1);
  return DZ_OK;
}

// Batched acting (parts.py:342-411 with many actors; dqn/agent.py:121-131,169-177): online forward on E <= batch observations
// in one enqueue, q-values [E][A], and the epsilon-greedy choice on the device — one D2H of E actions per tick instead of a
// D2H sync per decision.  E = 1 with d_actions NULL is select_action's network half.
int dz_learner_act_batch(dz_learner* l, const uint8_t* d_obs, int32_t E, const float* d_taus, const float* d_noise,
                         int64_t noise_ld, const float* d_explore, float epsilon, float* d_q_out, int32_t* d_actions,
                         void* stream) {
  if (E < 1 || E > l->B) return fail(DZ_EINVAL, "act_batch: 1 <= E <= learner batch");
  DZ_TRY(l->side.join(stream));   // pending side-stream work (asynchronous randomness)
  const ActTarget t{l, l->buf.d_online, learner_bufs(l), l->rows_act, nullptr, false, nullptr, l->fq_act_hat, l->fq_act_w};
  return act(t, E, d_obs, d_taus, d_noise, noise_ld, d_explore, epsilon, d_q_out, d_actions, stream);
}

int dz_learner_noise_stride(const dz_learner_config* cfg, int64_t* out) {
  DZ_TRY(validate(*cfg));
  if (!noisy_net(*cfg)) return fail(DZ_EINVAL, "noise_stride: only rainbow and noisy networks have noisy layers");
  *out = noise_layout(*cfg, make_dims(*cfg)).stride;
  return DZ_OK;
}

// E noise applies for dz_learner_act_batch's per-stream noise: the generator of dz_learner_generate_randomness over
// E * stride floats, so the first three applies equal what that call writes for the same seed and counter.  Advances
// the counter once.
int dz_learner_generate_stream_noise(dz_learner* l, uint64_t seed, int32_t E, float* d_noise, void* stream) {
  if (!noisy_net(l->cfg)) return fail(DZ_EINVAL, "generate_stream_noise: only rainbow and noisy networks have noisy layers");
  if (E < 1 || E > l->B) return fail(DZ_EINVAL, "generate_stream_noise: 1 <= E <= learner batch");
  if (!d_noise) return fail(DZ_EINVAL, "generate_stream_noise: null buffer");
  return launch_acting_draw(d_noise, (long long)E * noise_layout(l->cfg, l->d).stride, false, seed, l->buf.d_counters, stream);
}

// ------------------------------------------------------------------------------------------------
// Acting context: batched acting for up to kActorMaxStreams streams over the learner's online parameters, read in
// place (an act enqueued after a learner step on the same stream sees that step's parameters).  Its buffers are sized
// for its stream count; the torso and the 3136 -> 512 layer run on a forward-only tensor-core plan where the geometry
// allows it.
//
// A frozen actor (dz_actor_create_frozen) acts on a parameter snapshot of its own instead: P floats in the learner's
// layout inside its workspace, loaded by dz_actor_load_params, which also packs the conv weight images once.  It draws
// its randomness from a counter of its own, and its `l` is a shape-only learner (configuration, layout, offsets, dims
// and split counts; every device pointer NULL), so its act and randomness paths read and write nothing but its
// workspace, the caller's buffers and its plan's constant tables.
// ------------------------------------------------------------------------------------------------

struct dz_actor {
  dz_learner* l;               // live: the learner; frozen: a shape-only learner the actor owns
  int E;                       // streams
  NetBufs b;                   // activation set / head pass 1, as the learner's act_batch
  const uint8_t** rows;        // [E] observation row table
  float* noise;                // rainbow: the apply the tensor-core noisy1 reads (a copy of the caller's shared apply)
  UmNet* um;                   // forward-only tensor-core plan (nullptr: fp32-FMA torso)
  char* um_ws;
  bool frozen = false;
  bool loaded = false;         // frozen: dz_actor_load_params has run
  float* params = nullptr;     // frozen: the parameter snapshot, [P] in the learner's layout
  float* frac_hat = nullptr;   // fqf: the acting pass's tau_hat and interval weights, [E][N] each
  float* frac_w = nullptr;
  int64_t* counters = nullptr; // frozen: [2]; [1] is the generator counter (the slot randomness_kernel reads)
};

namespace {

constexpr int kActorMaxStreams = 1024, kActorMaxIqnRows = 16384;

// Rows per observation of the acting pass of iqn's network: the policy taus, or fqf's N fractions.
int acting_samples(const dz_learner_config& c) { return proposes_fractions(c.kind) ? c.num_fractions : c.tau_samples_policy; }

int actor_check(const dz_learner_config& c, int E) {
  if (E < 1 || E > kActorMaxStreams) return fail(DZ_EINVAL, "actor: num_streams must be in [1, 1024]");
  if (draws_taus(c.kind) && (int64_t)E * c.tau_samples_policy > kActorMaxIqnRows)
    return fail(DZ_EINVAL, "actor: num_streams * tau_samples_policy must be <= 16384");
  if (proposes_fractions(c.kind) && (int64_t)E * c.num_fractions > kActorMaxIqnRows)
    return fail(DZ_EINVAL, "actor: num_streams * num_fractions must be <= 16384");
  return DZ_OK;
}

// online: the parameter blob the plan's conv / fc tensor maps, bias reads and weight packing use.
UmNetDesc actor_um_desc(const dz_learner* l, int E, const float* online) {
  UmNetDesc u = make_um_desc(l);
  u.B = E; u.npass = 1; u.fwd_only = 1;
  u.online = online;
  u.pass_target[0] = 0; u.target = nullptr;
  for (int p = 0; p < 3; ++p) u.noise_apply[p] = 0;
  return u;
}

// Carves the actor's buffers (sizes only when base is NULL); the tensor-core plan's own buffers come from um_ws.
int64_t carve_actor(dz_actor* a, const dz_learner* l, char* base) {
  const dz_learner_config& c = l->cfg;
  const Dims& d = l->d;
  const int E = a->E;
  const FcNet& f = l->fc;
  const bool iqn = uses_iqn_net(c.kind);
  Bump w{base};
  NetBufs& b = a->b;
  memset(&b, 0, sizeof(b));   // split_rows 0: the fp32 GEMMs never split K, so row e's sums do not depend on E
  const UmNetDesc ud = actor_um_desc(l, E, nullptr);   // sizes only
  const bool um = um_net_supported(ud);
  a->um_ws = um ? w.take<char>(um_net_workspace_bytes(ud)) : nullptr;
  if (!um) {
    b.act1[1] = w.take<float>((int64_t)E * d.h1 * d.w1 * 32);
    b.act2[1] = w.take<float>((int64_t)E * d.h2 * d.w2 * 64);
    b.act3[1] = w.take<float>((int64_t)E * d.feat);
    b.conv_partial = w.take<float>((int64_t)l->conv_splits * E * d.h2 * d.w2 * 64);
  }
  const int64_t rows = (int64_t)E * (iqn ? acting_samples(c) : 1);
  if (!um || iqn) {                      // otherwise h1 is the tensor-core plan's
    b.h1[1][0] = w.take<float>(rows * 512);
    b.h1[1][1] = f.ns == 2 ? w.take<float>(rows * 512) : nullptr;
  }
  b.out[1] = w.take<float>(rows * d.out);
  b.outv[1] = f.ns == 2 && !f.dueling_head ? w.take<float>((int64_t)E * f.out[1]) : nullptr;
  b.cosf[1] = iqn ? w.take<float>(rows * c.latent_dim) : nullptr;
  b.hi[1] = iqn ? w.take<float>(rows * d.feat) : nullptr;
  a->rows = w.take<const uint8_t*>(E);
  a->noise = noisy_net(c) ? w.take<float>(noise_layout(c, d).stride) : nullptr;
  a->frac_hat = proposes_fractions(c.kind) ? w.take<float>((int64_t)E * c.num_fractions) : nullptr;
  a->frac_w = proposes_fractions(c.kind) ? w.take<float>((int64_t)E * c.num_fractions) : nullptr;
  if (a->frozen) {
    a->params = w.take<float>(l->lay.total);
    a->counters = w.take<int64_t>(2);
  }
  return w.used;
}

int actor_plan_bytes(const dz_learner_config* cfg, int32_t num_streams, bool frozen, int64_t* workspace_bytes) {
  if (!cfg || !workspace_bytes) return fail(DZ_EINVAL, "actor plan query: null argument");
  DZ_TRY(validate(*cfg));
  DZ_TRY(actor_check(*cfg, num_streams));
  dz_learner tmp;
  init_shape_learner(&tmp, *cfg);
  dz_actor a;
  a.E = num_streams;
  a.frozen = frozen;
  *workspace_bytes = carve_actor(&a, &tmp, nullptr);
  return DZ_OK;
}

// l: the learner (live) or a shape-only learner the actor takes over (frozen).
int actor_create(dz_learner* l, bool frozen, int32_t num_streams, void* d_workspace, dz_actor** out) {
  dz_actor* a = new dz_actor();
  a->l = l;
  a->E = num_streams;
  a->frozen = frozen;
  carve_actor(a, l, static_cast<char*>(d_workspace));
  if (frozen) {
    cudaError_t e = cudaMemsetAsync(a->counters, 0, 2 * sizeof(int64_t), 0);
    if (e == cudaSuccess) e = cudaStreamSynchronize(0);
    if (e != cudaSuccess) { dz_actor_destroy(a); return fail(DZ_ECUDA, "frozen actor: counter init: %s", cudaGetErrorString(e)); }
  }
  if (a->um_ws) {
    int rc = um_net_create(actor_um_desc(l, num_streams, frozen ? a->params : l->buf.d_online), a->um_ws, &a->um);
    if (rc == DZ_OK && a->noise) rc = um_bind_noise(a->um, a->noise);
    if (rc != DZ_OK) { dz_actor_destroy(a); return rc; }
    for (int L = 1; L <= 3; ++L) (L == 1 ? a->b.act1 : L == 2 ? a->b.act2 : a->b.act3)[1] = um_act_f32(a->um, L, 0);
    if (!uses_iqn_net(l->cfg.kind))
      for (int s = 0; s < l->fc.ns; ++s) a->b.h1[1][s] = um_h1_f32(a->um, 0, s);
  }
  *out = a;
  return DZ_OK;
}

}  // namespace

int dz_actor_plan_query(const dz_learner_config* cfg, int32_t num_streams, int64_t* workspace_bytes) {
  return actor_plan_bytes(cfg, num_streams, false, workspace_bytes);
}

int dz_actor_frozen_plan_query(const dz_learner_config* cfg, int32_t num_streams, int64_t* workspace_bytes) {
  return actor_plan_bytes(cfg, num_streams, true, workspace_bytes);
}

int dz_actor_create(dz_learner* l, int32_t num_streams, void* d_workspace, dz_actor** out) {
  if (!l || !d_workspace || !out) return fail(DZ_EINVAL, "actor create: null argument");
  DZ_TRY(actor_check(l->cfg, num_streams));
  return actor_create(l, false, num_streams, d_workspace, out);
}

int dz_actor_create_frozen(dz_learner* l, int32_t num_streams, void* d_workspace, dz_actor** out) {
  if (!l || !d_workspace || !out) return fail(DZ_EINVAL, "frozen actor create: null argument");
  DZ_TRY(actor_check(l->cfg, num_streams));
  dz_learner* shape = new dz_learner();
  init_shape_learner(shape, l->cfg);
  return actor_create(shape, true, num_streams, d_workspace, out);   // on failure the actor's destroy frees shape
}

void dz_actor_destroy(dz_actor* a) {
  if (!a) return;
  um_net_destroy(a->um);
  if (a->frozen) delete a->l;
  delete a;
}

// Frozen actor: snapshot <- d_src (a full parameter blob in the learner's layout, e.g. its online blob), then the conv
// weight images of the tensor-core plan are packed from the snapshot, once.  Both are enqueued on `stream`.
int dz_actor_load_params(dz_actor* a, const float* d_src, void* stream) {
  if (!a || !d_src) return fail(DZ_EINVAL, "actor load_params: null argument");
  if (!a->frozen) return fail(DZ_EINVAL, "load_params: a live actor reads the learner's parameters in place (create a frozen actor)");
  DZ_CUDA_OK(cudaMemcpyAsync(a->params, d_src, a->l->lay.total * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  if (a->um) DZ_TRY(um_pack_weights(a->um, stream));
  a->loaded = true;
  return DZ_OK;
}

// Frozen actor: d_dst <- the snapshot (P floats), enqueued on `stream`.
int dz_actor_get_params(dz_actor* a, float* d_dst, void* stream) {
  if (!a || !d_dst) return fail(DZ_EINVAL, "actor get_params: null argument");
  if (!a->frozen || !a->loaded) return fail(DZ_EINVAL, "get_params: the actor holds no parameter snapshot");
  DZ_CUDA_OK(cudaMemcpyAsync(d_dst, a->params, a->l->lay.total * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return DZ_OK;
}

// Frozen actor: its generator counter, read after the work enqueued on `stream` (which this call waits for).
int dz_actor_get_counter(dz_actor* a, int64_t* out, void* stream) {
  if (!a || !out) return fail(DZ_EINVAL, "actor get_counter: null argument");
  if (!a->frozen) return fail(DZ_EINVAL, "get_counter: a live actor advances the learner's counter");
  int64_t v = 0;
  DZ_CUDA_OK(cudaMemcpyAsync(&v, a->counters + 1, sizeof(int64_t), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  DZ_CUDA_OK(cudaStreamSynchronize((cudaStream_t)stream));
  *out = v;
  return DZ_OK;
}

// Frozen actor: sets its generator counter, ordered on `stream` (the call returns once the value is staged).
int dz_actor_set_counter(dz_actor* a, int64_t value, void* stream) {
  if (!a) return fail(DZ_EINVAL, "actor set_counter: null handle");
  if (!a->frozen) return fail(DZ_EINVAL, "set_counter: a live actor advances the learner's counter");
  DZ_CUDA_OK(cudaMemcpyAsync(a->counters + 1, &value, sizeof(int64_t), cudaMemcpyHostToDevice, (cudaStream_t)stream));
  DZ_CUDA_OK(cudaStreamSynchronize((cudaStream_t)stream));
  return DZ_OK;
}

// dz_learner_act_batch's contract for the actor's num_streams observations.  noise_ld (rainbow): 0, d_noise is one
// apply shared by every stream (noisy1 on the tensor cores when the torso is); the noise stride, d_noise is [E][stride]
// and stream e uses apply e (noisy layers on the per-row fp32 kernels).
int dz_actor_act(dz_actor* a, const uint8_t* d_obs, const float* d_taus, const float* d_noise, int64_t noise_ld,
                 const float* d_explore, float epsilon, float* d_q_out, int32_t* d_actions, void* stream) {
  if (!a) return fail(DZ_EINVAL, "actor: null handle");
  if (!d_actions) return fail(DZ_EINVAL, "actor: null buffer");
  if (a->frozen && !a->loaded) return fail(DZ_EINVAL, "frozen actor: no parameters loaded (dz_actor_load_params)");
  const ActTarget t{a->l, a->frozen ? a->params : a->l->buf.d_online, a->b, a->rows, a->um, !a->frozen, a->noise,
                    a->frac_hat, a->frac_w};
  return act(t, a->E, d_obs, d_taus, d_noise, noise_ld, d_explore, epsilon, d_q_out, d_actions, stream);
}

// The actor's randomness from the learner's generator and counter: iqn taus [E][tau_samples_policy] (the stream id of
// dz_learner_generate_randomness's taus); rainbow one noise apply, or E applies when per_stream is set (the stream id of
// its noise and of dz_learner_generate_stream_noise).  Advances d_counters[1] once.  A frozen actor draws the same way
// from its own counter and never touches the learner's.
int dz_actor_generate_randomness(dz_actor* a, uint64_t seed, int32_t per_stream, float* d_out, void* stream) {
  if (!a || !d_out) return fail(DZ_EINVAL, "actor randomness: null argument");
  const dz_learner_config& c = a->l->cfg;
  long long n;
  const bool iqn = draws_taus(c.kind);
  if (iqn && !per_stream) n = (long long)a->E * c.tau_samples_policy;
  else if (noisy_net(c)) n = (per_stream ? (long long)a->E : 1LL) * noise_layout(c, a->l->d).stride;
  else return fail(DZ_EINVAL, "actor randomness: iqn draws taus, noisy layers noise (per_stream: noise only); other kinds draw nothing");
  return launch_acting_draw(d_out, n, iqn, seed, a->frozen ? a->counters : a->l->buf.d_counters, stream);
}

// Test hook: the MMA path of the actor's tensor-core launch `tag` (the tags of dz_test_learner_mma_path's torso and fc
// launches).  DZ_EINVAL when the actor runs on the fp32-FMA kernels or has no such launch.
int dz_test_actor_mma_path(dz_actor* a, const char* tag, int32_t* path) {
  if (!a->um) return fail(DZ_EINVAL, "the actor runs on the fp32-FMA kernels (geometry outside the tensor-core path)");
  const int p = um_net_mma_path(a->um, tag);
  if (p < 0) return fail(DZ_EINVAL, "no tensor-core launch '%s' in this actor", tag ? tag : "");
  *path = p;
  return DZ_OK;
}

// Test hook: device pointer + element count of the actor's conv3 output "act3" ([E][feat], written by the last act).
int dz_test_actor_buffer(dz_actor* a, const char* name, float** d_ptr, int64_t* count) {
  if (std::string(name ? name : "") != "act3") return fail(DZ_EINVAL, "unknown actor buffer '%s'", name ? name : "");
  *d_ptr = a->b.act3[1];
  *count = (int64_t)a->E * a->l->d.feat;
  return DZ_OK;
}

namespace {
__global__ void u8_to_unit_table_kernel(float* out) {
  dz::pdl_enter();
  out[threadIdx.x] = u8_to_unit(threadIdx.x);
}
}  // namespace

// Test hook: the device's uint8 -> float32/255 conversion of 0..255 (the conv1 operand load of the fp32-FMA kernels).
int dz_test_u8_to_unit(float* d_out256, void* stream) {
  DZ_LAUNCH(u8_to_unit_table_kernel, 1, 256, 0, stream, d_out256);
  return DZ_OK;
}

int dz_learner_sync_target(dz_learner* l, void* stream) {
  DZ_CUDA_OK(cudaMemcpyAsync(l->buf.d_target, l->buf.d_online, l->lay.total * sizeof(float), cudaMemcpyDeviceToDevice,
                             (cudaStream_t)stream));
  return DZ_OK;
}

// Debug hook: the tensor-core launch named `tag` ("conv1_fwd", "conv2_fwd", "conv3_fwd", "fc1_fwd", "fc1_dgrad", "conv3_dgrad",
// "conv2_dgrad", "conv3_wgrad", "conv2_wgrad") writes the clock stamps of its CTA 0 into d_trace (512 int64); nullptr switches
// it off.  conv1_fwd stamps per output tile, the others per shared-memory stage (tools/umma_stage_trace.py reads both).
int dz_test_learner_trace(dz_learner* l, const char* tag, long long* d_trace) {
  if (!l->um) return fail(DZ_EINVAL, "the tensor-core path is not active for this learner");
  um_net_trace(l->um, tag, d_trace);
  return DZ_OK;
}

// Test hook: the MMA path of the tensor-core launch named `tag` (the tags of dz_test_learner_trace, conv1_fwd included):
// 1 warp-level mma.sync kernel, 2 wgmma kernel.  The IQN update's launches "iqn_embed_fwd", "iqn_fc1_fwd",
// "iqn_fc1_wgrad", "iqn_fc1_dgrad" and "iqn_embed_wgrad" answer 1 when they run on the packed-operand GEMM
// (tc_pgemm_kernel) and DZ_EINVAL when they run on the fp32-FMA kernels, whatever path the torso takes.
int dz_test_learner_mma_path(dz_learner* l, const char* tag, int32_t* path) {
  const std::string t = tag ? tag : "";
  if (t == "iqn_embed_fwd" || t == "iqn_fc1_fwd" || t == "iqn_fc1_wgrad" || t == "iqn_fc1_dgrad" || t == "iqn_embed_wgrad") {
    const bool packed = l->pk_on && (t != "iqn_embed_wgrad" || l->pk_embed_bwd);
    if (!packed) return fail(DZ_EINVAL, "'%s' does not run on the packed tensor-core GEMM in this learner", tag);
    *path = UM_PATH_MMA_SYNC;
    return DZ_OK;
  }
  if (!l->um) return fail(DZ_EINVAL, "the tensor-core path is not active for this learner");
  const int p = um_net_mma_path(l->um, tag);
  if (p < 0) return fail(DZ_EINVAL, "no tensor-core launch '%s' in this learner", tag ? tag : "");
  *path = p;
  return DZ_OK;
}

// Test hook: device-to-device copy out of an internal buffer (tests hold only the raw pointer).
int dz_test_copy(void* d_dst, const void* d_src, int64_t bytes, void* stream) {
  DZ_CUDA_OK(cudaMemcpyAsync(d_dst, d_src, (size_t)bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return DZ_OK;
}

int dz_test_random_shift(const uint8_t* const* d_rows_tm1, const uint8_t* const* d_rows_t, const int32_t* d_shifts,
                         int32_t B, int32_t H, int32_t W, int32_t C, int32_t pad, uint8_t* d_out, int64_t out_stride,
                         void* stream) {
  if (!d_rows_tm1 || !d_rows_t || !d_shifts || !d_out) return fail(DZ_EINVAL, "random_shift: null buffer");
  if (B < 1 || B > 65535 || H < 1 || W < 1 || C < 4 || C % 4) return fail(DZ_EINVAL, "random_shift: bad B / H / W / C");
  if (pad < 0 || pad > kShiftMaxPad || pad >= std::min(H, W)) return fail(DZ_EINVAL, "random_shift: pad must be in [0,16] and < min(H, W)");
  const int64_t row = (int64_t)W * C;
  if (row % 16 || row > kShiftStageBytes) return fail(DZ_EINVAL, "random_shift: W * C must be a multiple of 16 and at most 32768");
  if (out_stride < row * H || out_stride % 16 || (reinterpret_cast<uintptr_t>(d_out) & 15))
    return fail(DZ_EINVAL, "random_shift: out_stride must be >= H*W*C and a multiple of 16, d_out 16-byte aligned");
  return launch_random_shift(d_rows_tm1, d_rows_t, d_shifts, B, H, W, C, pad, d_out, out_stride, nullptr, nullptr, stream);
}

// Host twin of loss_munchausen_kernel's per-example arithmetic: the warp's xor-butterfly reductions over an array of 32
// lanes, then the same munchausen_exp / munchausen_target (tests only).
int dz_test_munchausen_example(const float* q_tm1, const float* qbar_tm1, const float* qbar_t, int32_t A, int32_t a_tm1,
                               float r_t, float discount_t, float alpha, float tau, float l0, float* out) {
  if (!q_tm1 || !qbar_tm1 || !qbar_t || !out) return fail(DZ_EINVAL, "munchausen example: NULL buffer");
  if (A < 1 || A > kMunchausenMaxActions || a_tm1 < 0 || a_tm1 >= A) return fail(DZ_EINVAL, "munchausen example: A or a_tm1 out of range");
  if (!munchausen_params_ok(alpha, tau, l0)) return fail(DZ_EINVAL, "munchausen example: bad alpha / tau / l0");
  auto butterfly = [](float* v, bool is_max) {
    for (int o = 16; o > 0; o >>= 1) {
      float t[32];
      for (int i = 0; i < 32; ++i) t[i] = is_max ? fmaxf(v[i], v[i ^ o]) : v[i] + v[i ^ o];
      for (int i = 0; i < 32; ++i) v[i] = t[i];
    }
    return v[0];
  };
  float red[2][2];   // [s_tm1, s_t][max, sum]
  const float* q[2] = {qbar_tm1, qbar_t};
  for (int s = 0; s < 2; ++s) {
    float v[32];
    for (int i = 0; i < 32; ++i) v[i] = i < A ? q[s][i] : -INFINITY;
    red[s][0] = butterfly(v, true);
    for (int i = 0; i < 32; ++i) v[i] = i < A ? munchausen_exp(q[s][i], red[s][0], tau) : 0.f;
    red[s][1] = butterfly(v, false);
  }
  const MunchausenTarget m = munchausen_target(r_t, discount_t, qbar_tm1[a_tm1], red[0][0], red[0][1], red[1][0], red[1][1],
                                               alpha, tau, l0);
  out[0] = m.target;
  out[1] = m.target - q_tm1[a_tm1];
  out[2] = m.bonus;
  return DZ_OK;
}

// Host twin of loss_munchausen_iqn_kernel's per-example target arithmetic: the same miqn_mean sums, the warp's
// xor-butterfly reductions over an array of 32 lanes, then the same munchausen_exp / miqn_h / munchausen_bonus /
// miqn_target (tests only).
int dz_test_munchausen_iqn_example(const float* zbar_tm1, const float* zbar_t, int32_t A, int32_t K, int32_t Nt,
                                   int32_t a_tm1, float r_t, float discount_t, float alpha, float tau, float l0, float* out) {
  if (!zbar_tm1 || !zbar_t || !out) return fail(DZ_EINVAL, "munchausen_iqn example: NULL buffer");
  if (A < 1 || A > kMunchausenMaxActions || a_tm1 < 0 || a_tm1 >= A || K < 1 || K > 256 || Nt < 1 || Nt > 256)
    return fail(DZ_EINVAL, "munchausen_iqn example: A, K, Nt or a_tm1 out of range");
  if (!munchausen_params_ok(alpha, tau, l0)) return fail(DZ_EINVAL, "munchausen_iqn example: bad alpha / tau / l0");
  auto butterfly = [](const float* in, bool is_max) {
    float v[32];
    for (int i = 0; i < 32; ++i) v[i] = in[i];
    for (int o = 16; o > 0; o >>= 1) {
      float t[32];
      for (int i = 0; i < 32; ++i) t[i] = is_max ? fmaxf(v[i], v[i ^ o]) : v[i] + v[i ^ o];
      for (int i = 0; i < 32; ++i) v[i] = t[i];
    }
    return v[0];
  };
  float q[2][32], lane[32];
  for (int a = 0; a < 32; ++a) {
    q[0][a] = a < A ? miqn_mean(zbar_tm1, K, A, a) : -INFINITY;
    q[1][a] = a < A ? miqn_mean(zbar_t, Nt, A, a) : -INFINITY;
  }
  const float v1 = butterfly(q[0], true), v2 = butterfly(q[1], true);
  for (int a = 0; a < 32; ++a) lane[a] = a < A ? munchausen_exp(q[0][a], v1, tau) : 0.f;
  const float s1 = butterfly(lane, false);
  float e2[32], pi[32];
  for (int a = 0; a < 32; ++a) e2[a] = a < A ? munchausen_exp(q[1][a], v2, tau) : 0.f;
  const float s2 = butterfly(e2, false);
  for (int a = 0; a < 32; ++a) pi[a] = e2[a] / s2;
  for (int a = 0; a < 32; ++a) lane[a] = a < A ? pi[a] * miqn_h(q[1][a], v2, s2, tau) : 0.f;
  const float ent = butterfly(lane, false);
  const float bonus = munchausen_bonus(q[0][a_tm1], v1, s1, alpha, tau, l0);
  for (int j = 0; j < Nt; ++j) out[j] = miqn_target(zbar_t + (long long)j * A, pi, A, r_t + bonus, discount_t, ent);
  out[Nt] = bonus;
  out[Nt + 1] = ent;
  return DZ_OK;
}

// Host twin of fqf's per-example fraction arithmetic: fqf_fractions and fqf_dlogits, the functions the fraction and
// loss kernels run (tests only).
int dz_test_fqf_example(const float* logits, const float* F_tau, const float* F_hat, int32_t N, float cot, float* out) {
  if (!logits || !F_tau || !F_hat || !out) return fail(DZ_EINVAL, "fqf example: NULL buffer");
  if (N < 2 || N > kFqfMaxFractions) return fail(DZ_EINVAL, "fqf example: N must be in [2,128]");
  float* q = out;
  float* tau = q + N;
  float* hat = tau + N + 1;
  float* w = hat + N;
  float* dl = w + N;
  fqf_fractions(logits, N, q, tau, hat, w);
  fqf_dlogits(F_tau, F_hat, q, N, cot, dl);
  return DZ_OK;
}

// Host twin of the dueling head's per-row arithmetic: dueling_aggregate and dueling_transpose, the functions
// dueling_head_fwd_kernel and dueling_head_bwd_kernel run (tests only).
int dz_test_dueling_example(const float* adv, float v, const float* dq, int32_t A, float* out) {
  if (!adv || !dq || !out) return fail(DZ_EINVAL, "dueling example: NULL buffer");
  if (A < 1 || A > kDuelingMaxActions) return fail(DZ_EINVAL, "dueling example: A must be in [1,64]");
  dueling_aggregate(adv, v, A, out);
  out[2 * A] = dueling_transpose(dq, A, out + A);
  return DZ_OK;
}

// Host twin of every loss kernel's CQL arithmetic: cql_example, the function their cql variants run (tests only).
int dz_test_cql_example(const float* q, int32_t A, int32_t a_tm1, float cot, float* out) {
  if (!q || !out) return fail(DZ_EINVAL, "cql example: NULL buffer");
  if (A < 1 || A > 64) return fail(DZ_EINVAL, "cql example: A must be in [1,64]");
  if (a_tm1 < 0 || a_tm1 >= A) return fail(DZ_EINVAL, "cql example: a_tm1 out of range");
  out[A] = cql_example(q, A, a_tm1, cot, out);
  return DZ_OK;
}

// The body of dz_test_loss and dz_test_loss_fqf: the learner's loss section (launch_loss) on caller-owned head outputs,
// batch and output buffers, all on `stream`; fqf: its fraction buffers.  The observation fields of cfg play no part;
// they are replaced by a legal geometry before validate().
static int test_loss_section(const dz_learner_config* cfg, int32_t B, const float* const* d_out, const float* const* d_val,
                             const int32_t* d_a_tm1, const float* d_r_t, const float* d_discount_t, const float* d_weights,
                             const float* d_taus, float* d_dout, float* d_dval, float* d_per_example, float* d_priorities,
                             float* d_loss_terms, float* d_loss, float* d_max_seen, const FqfLossArgs* fqf, void* stream) {
  if (!cfg || !d_out) return fail(DZ_EINVAL, "test_loss: NULL argument");
  dz_learner_config c = *cfg;
  c.batch = B; c.obs_h = 84; c.obs_w = 84; c.obs_c = 4;
  DZ_TRY(validate(c));
  const bool rb = c.kind == DZ_RAINBOW;
  if (!d_out[0] || !d_out[1] || !d_out[2] || (rb && (!d_val || !d_val[0] || !d_val[1] || !d_val[2] || !d_dval)))
    return fail(DZ_EINVAL, "test_loss: head outputs of three passes are required (rainbow: and value streams)");
  if (!d_a_tm1 || !d_r_t || !d_discount_t || !d_dout || !d_per_example || !d_loss_terms || !d_loss)
    return fail(DZ_EINVAL, "test_loss: NULL buffer");
  if (draws_taus(c.kind) && !d_taus) return fail(DZ_EINVAL, "test_loss: iqn needs taus[B][tau_samples_s_tm1]");
  if (writes_priorities(c) && !d_priorities) return fail(DZ_EINVAL, "test_loss: this learner writes priorities");
  LossArgs L;
  memset(&L, 0, sizeof(L));
  L.out0 = d_out[0]; L.out1 = d_out[1]; L.out2 = d_out[2];
  L.adv0 = d_out[0]; L.adv1 = d_out[1]; L.adv2 = d_out[2];
  if (rb) { L.val0 = d_val[0]; L.val1 = d_val[1]; L.val2 = d_val[2]; }
  L.a = d_a_tm1; L.r = d_r_t; L.disc = d_discount_t; L.w = d_weights; L.taus0 = d_taus;
  L.dout = d_dout; L.dadv = d_dout; L.dval = d_dval;
  L.per_example = d_per_example; L.loss_terms = d_loss_terms; L.priorities = d_priorities;
  return launch_loss(c, L, B, stream, nullptr, d_loss, d_max_seen, nullptr, fqf);
}

// Test hook: the loss section of every kind but fqf, whose loss needs the fraction buffers of dz_test_loss_fqf.
int dz_test_loss(const dz_learner_config* cfg, int32_t B, const float* const* d_out, const float* const* d_val,
                 const int32_t* d_a_tm1, const float* d_r_t, const float* d_discount_t, const float* d_weights,
                 const float* d_taus, float* d_dout, float* d_dval, float* d_per_example, float* d_priorities,
                 float* d_loss_terms, float* d_loss, float* d_max_seen, void* stream) {
  return test_loss_section(cfg, B, d_out, d_val, d_a_tm1, d_r_t, d_discount_t, d_weights, d_taus, d_dout, d_dval,
                           d_per_example, d_priorities, d_loss_terms, d_loss, d_max_seen, nullptr, stream);
}

// Test hook: fqf's loss section (loss_fqf_kernel, then loss_mean_kernel) with the fraction buffers.
int dz_test_loss_fqf(const dz_learner_config* cfg, int32_t B, const float* const* d_out, const int32_t* d_a_tm1,
                     const float* d_r_t, const float* d_discount_t, const float* d_weights, const float* d_tau_hat,
                     const float* d_w_t, const float* d_q_tm1, float* d_dout, float* d_dlogits, float* d_per_example,
                     float* d_loss_terms, float* d_loss, void* stream) {
  if (!cfg || !proposes_fractions(cfg->kind)) return fail(DZ_EINVAL, "test_loss_fqf: the configuration is not fqf");
  if (!d_tau_hat || !d_w_t || !d_q_tm1 || !d_dlogits)
    return fail(DZ_EINVAL, "test_loss_fqf: tau_hat, w_t, q_tm1 and dlogits [B][num_fractions] are required");
  const FqfLossArgs fl{d_w_t, d_q_tm1, d_dlogits};
  return test_loss_section(cfg, B, d_out, nullptr, d_a_tm1, d_r_t, d_discount_t, d_weights, d_tau_hat, d_dout, nullptr,
                           d_per_example, nullptr, d_loss_terms, d_loss, nullptr, &fl, stream);
}

// The body of dz_test_q_values and dz_test_q_values_fqf: the acting tail (launch_q_values) on caller-owned head outputs
// of E observations; fqf: with the interval weights frac_w.
static int test_q_values_tail(const dz_learner_config* cfg, int32_t E, const float* d_out, const float* d_val,
                              const float* d_explore, float epsilon, float* d_q_out, int32_t* d_actions,
                              const float* d_frac_w, void* stream) {
  if (!cfg) return fail(DZ_EINVAL, "test_q_values: NULL config");
  dz_learner_config c = *cfg;
  c.obs_h = 84; c.obs_w = 84; c.obs_c = 4;
  DZ_TRY(validate(c));
  if (E < 1) return fail(DZ_EINVAL, "test_q_values: E must be >= 1");
  if (!d_out || !d_q_out || (c.kind == DZ_RAINBOW && !d_val)) return fail(DZ_EINVAL, "test_q_values: NULL buffer");
  return launch_q_values(c, E, d_out, d_val, d_explore, epsilon, d_q_out, d_actions, stream, d_frac_w);
}

// Test hook: the acting tail of every kind but fqf (dz_test_q_values_fqf).
int dz_test_q_values(const dz_learner_config* cfg, int32_t E, const float* d_out, const float* d_val, const float* d_explore,
                     float epsilon, float* d_q_out, int32_t* d_actions, void* stream) {
  return test_q_values_tail(cfg, E, d_out, d_val, d_explore, epsilon, d_q_out, d_actions, nullptr, stream);
}

// Test hook: fqf's acting tail (q_values_fqf_kernel, act_select_kernel) with the interval weights.
int dz_test_q_values_fqf(const dz_learner_config* cfg, int32_t E, const float* d_out, const float* d_frac_w,
                         const float* d_explore, float epsilon, float* d_q_out, int32_t* d_actions, void* stream) {
  if (!cfg || !proposes_fractions(cfg->kind)) return fail(DZ_EINVAL, "test_q_values_fqf: the configuration is not fqf");
  if (!d_frac_w) return fail(DZ_EINVAL, "test_q_values_fqf: NULL interval weights");
  return test_q_values_tail(cfg, E, d_out, nullptr, d_explore, epsilon, d_q_out, d_actions, d_frac_w, stream);
}

// Test hook: the fraction proposal (launch_fraction_forward) of an fqf learner's layout on caller-owned buffers.
int dz_test_fraction_forward(dz_learner* l, int32_t E, int32_t napp, const float* const* d_feat, const float* d_params,
                             float* const* d_tau, float* const* d_tau_hat, float* const* d_w, float* const* d_q,
                             float* d_pass1, float* d_pass2, void* stream) {
  if (!l || !d_feat || !d_params) return fail(DZ_EINVAL, "test_fraction_forward: NULL argument");
  if (!proposes_fractions(l->cfg.kind)) return fail(DZ_EINVAL, "test_fraction_forward: the learner is not fqf");
  if (E < 1 || napp < 1 || napp > 2) return fail(DZ_EINVAL, "test_fraction_forward: E >= 1 and napp in {1, 2}");
  FracArgs f;
  memset(&f, 0, sizeof(f));
  for (int a = 0; a < napp; ++a) {
    if (!d_feat[a]) return fail(DZ_EINVAL, "test_fraction_forward: NULL features");
    f.feat[a] = d_feat[a];
    if (d_tau) f.tau[a] = d_tau[a];
    if (d_tau_hat) f.tau_hat[a] = d_tau_hat[a];
    if (d_w) f.w[a] = d_w[a];
    if (d_q) f.q[a] = d_q[a];
  }
  f.pass1 = d_pass1; f.pass2 = d_pass2;
  return launch_fraction_forward(l, f, d_params, E, napp, stream);
}

// Test hook: the dueling head forward (launch_dueling_head_fwd) of a dueling learner's layout on caller-owned buffers.
int dz_test_dueling_head_fwd(dz_learner* l, int32_t rows, int32_t np, const float* const* d_h1, const float* const* d_params,
                             const float* const* d_noise, int64_t noise_ld, float* const* d_out, void* stream) {
  if (!l || !d_h1 || !d_params || !d_out) return fail(DZ_EINVAL, "test_dueling_head_fwd: NULL argument");
  const dz_learner_config& c = l->cfg;
  if (!l->fc.dueling_head) return fail(DZ_EINVAL, "test_dueling_head_fwd: the learner is not dueling");
  if (rows < 1 || np < 1 || np > 3 || noise_ld < 0) return fail(DZ_EINVAL, "test_dueling_head_fwd: rows, np or noise_ld out of range");
  if (noisy_net(c) ? !d_noise : noise_ld != 0) return fail(DZ_EINVAL, "test_dueling_head_fwd: noise only for the noisy network");
  const float* h1[3][2];
  for (int i = 0; i < np; ++i) {
    h1[i][0] = d_h1[2 * i]; h1[i][1] = d_h1[2 * i + 1];
    if (!h1[i][0] || !h1[i][1] || !d_params[i] || !d_out[i] || (d_noise && !d_noise[i]))
      return fail(DZ_EINVAL, "test_dueling_head_fwd: NULL buffer");
  }
  return launch_dueling_head_fwd(l, rows, np, h1, d_params, d_out, d_noise, noise_ld, stream);
}

// Test hook: the dueling head backward (launch_dueling_head_bwd) of a dueling learner's layout on caller-owned buffers.
int dz_test_dueling_head_bwd(dz_learner* l, int32_t rows, float* d_dq, float* d_dval, const float* const* d_h1,
                             const float* d_params, const float* d_noise, float* const* d_dh1, float* const* d_hi,
                             float* const* d_lo, void* stream) {
  if (!l || !d_dq || !d_dval || !d_h1 || !d_params || !d_dh1) return fail(DZ_EINVAL, "test_dueling_head_bwd: NULL argument");
  const dz_learner_config& c = l->cfg;
  if (!l->fc.dueling_head) return fail(DZ_EINVAL, "test_dueling_head_bwd: the learner is not dueling");
  if (rows < 1) return fail(DZ_EINVAL, "test_dueling_head_bwd: rows must be >= 1");
  if (noisy_net(c) && !d_noise) return fail(DZ_EINVAL, "test_dueling_head_bwd: the noisy network needs its noise apply");
  if (!d_h1[0] || !d_h1[1] || !d_dh1[0] || !d_dh1[1] || (!d_hi != !d_lo) || (d_hi && (!d_hi[0] || !d_hi[1] || !d_lo[0] || !d_lo[1])))
    return fail(DZ_EINVAL, "test_dueling_head_bwd: NULL buffer");
  return launch_dueling_head_bwd(l, rows, d_dq, d_dval, d_h1, d_params, d_dh1, d_hi, d_lo, d_noise, stream);
}

// Test hook: rainbow's noisy head forward (launch_noisy_head_fwd) of a rainbow learner's layout on caller-owned buffers.
int dz_test_noisy_head_fwd(dz_learner* l, int32_t rows, int32_t np, const float* const* d_h1, const float* const* d_params,
                           const float* d_noise, float* const* d_out, void* stream) {
  if (!l || !d_h1 || !d_params || !d_noise || !d_out) return fail(DZ_EINVAL, "test_noisy_head_fwd: NULL argument");
  if (np < 1 || np > 3) return fail(DZ_EINVAL, "test_noisy_head_fwd: np must be in 1..3");
  NetBufs nb;
  memset(&nb, 0, sizeof(nb));
  Pass passes[3];
  for (int i = 0; i < np; ++i) {
    if (!d_h1[2 * i] || !d_h1[2 * i + 1] || !d_params[i] || !d_out[2 * i] || !d_out[2 * i + 1])
      return fail(DZ_EINVAL, "test_noisy_head_fwd: NULL buffer");
    nb.h1[i][0] = const_cast<float*>(d_h1[2 * i]); nb.h1[i][1] = const_cast<float*>(d_h1[2 * i + 1]);
    nb.out[i] = d_out[2 * i]; nb.outv[i] = d_out[2 * i + 1];
    passes[i] = Pass{d_params[i], 0, i, i};
  }
  return launch_noisy_head_fwd(l, nb, passes, np, rows, d_noise, stream);
}

// Test hook: rainbow's noisy head input gradient (launch_noisy_head_bwd) on caller-owned buffers.
int dz_test_noisy_head_bwd(dz_learner* l, int32_t rows, const float* const* d_dout, const float* d_params, const float* d_noise,
                           const float* const* d_h1, float* const* d_dh1, float* const* d_hi, float* const* d_lo, void* stream) {
  if (!l || !d_dout || !d_params || !d_noise || !d_h1 || !d_dh1) return fail(DZ_EINVAL, "test_noisy_head_bwd: NULL argument");
  if ((!d_hi != !d_lo)) return fail(DZ_EINVAL, "test_noisy_head_bwd: hi and lo go together");
  float* none[2] = {nullptr, nullptr};
  return launch_noisy_head_bwd(l, rows, d_dout, d_params, d_noise, d_h1, d_dh1, d_hi ? d_hi : none, d_lo ? d_lo : none, stream);
}

// Test hook: IQN's cosine features (launch_iqn_cos) on caller-owned buffers.
int dz_test_iqn_cos(const float* d_taus, int64_t rows, int32_t latent, float* d_out, void* stream) {
  if (!d_taus || !d_out) return fail(DZ_EINVAL, "test_iqn_cos: NULL buffer");
  if (rows < 1 || latent < 1) return fail(DZ_EINVAL, "test_iqn_cos: rows and latent must be >= 1");
  return launch_iqn_cos(d_taus, d_out, rows, latent, stream);
}

static bool misaligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) != 0; }

// Test hook: IQN's value head (launch_iqn_head_fwd) of an IQN-network learner's layout on caller-owned buffers.
int dz_test_iqn_head_fwd(dz_learner* l, int32_t np, const int32_t* M, const float* const* d_h1, const float* const* d_params,
                         float* const* d_out, void* stream) {
  if (!l || !M || !d_h1 || !d_params || !d_out) return fail(DZ_EINVAL, "test_iqn_head_fwd: NULL argument");
  if (!uses_iqn_net(l->cfg.kind)) return fail(DZ_EINVAL, "test_iqn_head_fwd: the learner has no IQN network");
  if (l->d.out > kSkinnyMaxN) return fail(DZ_EINVAL, "test_iqn_head_fwd: the one-warp-per-row head takes at most 18 actions");
  if (np < 1 || np > 3) return fail(DZ_EINVAL, "test_iqn_head_fwd: np must be in [1, 3]");
  int m[3];
  for (int i = 0; i < np; ++i) {
    if (M[i] < 1) return fail(DZ_EINVAL, "test_iqn_head_fwd: M must be >= 1");
    if (!d_h1[i] || !d_params[i] || !d_out[i]) return fail(DZ_EINVAL, "test_iqn_head_fwd: NULL buffer");
    if (misaligned16(d_h1[i])) return fail(DZ_EINVAL, "test_iqn_head_fwd: h1 rows are read as float4");
    m[i] = M[i];
  }
  return launch_iqn_head_fwd(l, np, d_h1, d_params, d_out, m, stream);
}

// Test hook: the value head's input gradient (launch_iqn_head_dgrad) of an IQN-network learner's layout.
int dz_test_iqn_head_dgrad(dz_learner* l, int32_t M, const float* d_dout, const float* d_params, const float* d_h1,
                           float* d_dh1, void* stream) {
  if (!l || !d_dout || !d_params || !d_h1 || !d_dh1) return fail(DZ_EINVAL, "test_iqn_head_dgrad: NULL argument");
  if (!uses_iqn_net(l->cfg.kind)) return fail(DZ_EINVAL, "test_iqn_head_dgrad: the learner has no IQN network");
  if (l->d.out > kSkinnyMaxN) return fail(DZ_EINVAL, "test_iqn_head_dgrad: the kernel takes at most 18 actions");
  if (M < 1) return fail(DZ_EINVAL, "test_iqn_head_dgrad: M must be >= 1");
  if (misaligned16(d_h1) || misaligned16(d_dh1)) return fail(DZ_EINVAL, "test_iqn_head_dgrad: h1 and dh1 are accessed as float4");
  return launch_iqn_head_dgrad(l, d_dout, d_params, d_h1, d_dh1, M, stream);
}

// Test hook: the backward of IQN's Hadamard product (launch_iqn_hadamard_bwd), unpacked or packed.
int dz_test_iqn_hadamard_bwd(int32_t packed, int32_t B, int32_t N, int32_t D, float* d_dhi, const float* d_E, const float* d_F,
                             float* d_dfeat, float* d_img_hi, float* d_img_lo, int32_t img_rows_pad, void* stream) {
  if (!d_dhi || !d_E || !d_F || !d_dfeat) return fail(DZ_EINVAL, "test_iqn_hadamard_bwd: NULL buffer");
  if (B < 1 || N < 1 || D < 1) return fail(DZ_EINVAL, "test_iqn_hadamard_bwd: B, N and D must be >= 1");
  if (packed) {
    if (N != 64 || D % 64) return fail(DZ_EINVAL, "test_iqn_hadamard_bwd: the packed kernel needs N = 64 and D % 64 = 0");
    if (!d_img_hi || !d_img_lo || img_rows_pad % 128 || img_rows_pad < D)
      return fail(DZ_EINVAL, "test_iqn_hadamard_bwd: the packed kernel writes a [rows_pad >= D][B * 64] image");
    if (misaligned16(d_dhi) || misaligned16(d_E) || misaligned16(d_F) || misaligned16(d_img_hi) || misaligned16(d_img_lo))
      return fail(DZ_EINVAL, "test_iqn_hadamard_bwd: the packed kernel accesses its buffers as float4");
  }
  return launch_iqn_hadamard_bwd(packed != 0, d_dhi, d_E, d_F, d_dfeat, d_img_hi, d_img_lo, img_rows_pad / 8, B, N, D, stream);
}

// Test hook: device pointer + element count of an internal activation / gradient buffer (tests and tools only).
int dz_test_learner_buffer(dz_learner* l, const char* name, float** d_ptr, int64_t* count) {
  const std::string n = name;
  const int64_t rows0 = (int64_t)l->B * l->n_head[0];
  if (n == "act3") { *d_ptr = l->act3[0]; *count = (int64_t)l->B * l->d.feat; }
  else if (n == "act1") { *d_ptr = l->act1[0]; *count = (int64_t)l->B * l->d.h1 * l->d.w1 * 32; }
  else if (n == "act2") { *d_ptr = l->act2[0]; *count = (int64_t)l->B * l->d.h2 * l->d.w2 * 64; }
  else if (n == "h1_val") { *d_ptr = l->h1[0][1]; *count = l->h1[0][1] ? rows0 * 512 : 0; }
  else if (n == "iqn_e0") { *d_ptr = l->E0; *count = l->E0 ? rows0 * l->d.feat : 0; }
  else if (n == "h1") { *d_ptr = l->h1[0][0]; *count = rows0 * 512; }
  else if (n == "out0" || n == "out1" || n == "out2") {   // head pass p's outputs
    const int p = n[3] - '0';
    *d_ptr = l->out[p]; *count = (int64_t)l->B * l->n_head[p] * l->d.out;
  }
  else if (n == "dh1") { *d_ptr = l->dh1[0]; *count = rows0 * 512; }
  else if (n == "dh1_val") { *d_ptr = l->dh1[1]; *count = l->dh1[1] ? rows0 * 512 : 0; }
  else if (n == "dact1" || n == "dact2" || n == "dact3" || n == "dact1_hi" || n == "dact2_hi" || n == "dact3_hi" ||
           n == "dact1_lo" || n == "dact2_lo" || n == "dact3_lo" || n == "act1_lo" || n == "act2_lo") {
    const bool act = n[1] == 'c';   // "act1_lo", "act2_lo"
    const int layer = n[act ? 3 : 4] - '0';
    const int64_t per[3] = {(int64_t)l->B * l->d.h1 * l->d.w1 * 32, (int64_t)l->B * l->d.h2 * l->d.w2 * 64,
                            (int64_t)l->B * l->d.feat};
    float* f32[3] = {l->dact1, l->dact2, l->dact3};
    if (n.size() == (act ? 4u : 5u)) *d_ptr = f32[layer - 1];
    else if (!l->um) return fail(DZ_EINVAL, "%s is not materialised on the fp32-FMA torso", name);
    else *d_ptr = act ? um_act_lo(l->um, layer) : n.back() == 'i' ? um_dact_hi(l->um, layer) : um_dact_lo(l->um, layer);
    *count = per[layer - 1];
  }
  else if (n == "iqn_hi") {
    if (l->pk_on) return fail(DZ_EINVAL, "iqn_hi is not materialised on the packed tensor-core path");
    *d_ptr = l->hi[0]; *count = l->hi[0] ? rows0 * l->d.feat : 0;
  }
  else if (n == "iqn_dhi") { *d_ptr = l->dhi; *count = l->dhi ? rows0 * l->d.feat : 0; }
  else if (n == "fqf_tau") { *d_ptr = l->fq_tau; *count = (int64_t)2 * l->B * (l->cfg.num_fractions + 1); }
  else if (n == "fqf_tau_hat") { *d_ptr = l->fq_hat; *count = (int64_t)2 * l->B * l->cfg.num_fractions; }
  else if (n == "fqf_dlogits") { *d_ptr = l->fq_dlogits; *count = (int64_t)l->B * l->cfg.num_fractions; }
  else return fail(DZ_EINVAL, "unknown buffer '%s'", name);
  if (!*d_ptr) return fail(DZ_EINVAL, "buffer '%s' is not used by this agent kind", name);
  return DZ_OK;
}

}  // extern "C"
