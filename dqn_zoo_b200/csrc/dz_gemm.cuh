// Grouped fp32 GEMM kernels for the learner (SIMT path: exact-fp32 products, fp32 accumulate).
//
// Every layer of the Nature-CNN family is expressed as one of three contractions over a small
// table of problems (one launch covers all forward passes / streams of that layer):
//
//   NN  C[M,N]  = A[M,K]  * B[K,N]      forward (A = activations or implicit im2col, B = weights)
//   TN  C[K,N]  = A[M,K]^T * G[M,N]     weight gradient (reduction over the batch*spatial dim M)
//   NT  C[M,K]  = G[M,N]  * B[K,N]^T    input gradient  (reduction over N)
//
// A can be (i) a dense row-major matrix, (ii) an implicit im2col view of an NHWC float tensor or
// (iii) an implicit im2col view of uint8 observation rows addressed through a pointer table —
// the replay gather is fused here: conv1 reads sampled transitions in place, converting
// uint8 -> float32 / 255 on the fly (networks.py:193).  Weight layouts follow haiku: conv HWIO
// == row-major [KH*KW*Cin, Cout], linear [in, out] (networks_test.py:44,53).
#pragma once
#include "dz_common.cuh"

namespace dz {

enum : int { A_PLAIN = 0, A_CONV_F32 = 1, A_CONV_U8 = 2 };

// Division by a runtime constant without the integer-divide sequence: q = (umulhi(n, mul) + n) >> shr
// (round-up method, exact for 0 <= n < 2^31); initialised on the host.
struct FastDiv {
  uint32_t mul, shr;
  int d;
};
inline FastDiv make_fastdiv(int d) {
  FastDiv f;
  f.d = d < 1 ? 1 : d;
  uint32_t s = 0;
  while ((1u << s) < (uint32_t)f.d) ++s;
  f.shr = s;
  f.mul = (uint32_t)((((uint64_t)1 << 32) * (((uint64_t)1 << s) - (uint64_t)f.d)) / (uint64_t)f.d + 1);
  return f;
}
__device__ __forceinline__ int fd_div(int n, const FastDiv& f) {
  return (int)(((uint32_t)__umulhi((uint32_t)n, f.mul) + (uint32_t)n) >> f.shr);
}


struct GemmProblem {
  const void* A;        // A_PLAIN/A_CONV_F32: const float*;  A_CONV_U8: const uint8_t* const* (row table)
  const float* B;       // NN/NT: weights [K,N];  TN: G [M,N]
  const float* B2;      // dual (noisy) second weight matrix (sigma) or nullptr
  float* C;
  float* C2;            // second output (NN: pre-multiply activation E for IQN; TN: sigma-weight grad)
  int M, N, K;
  int lda, ldb, ldc;
  int a_mode;
  int H, W, Cin, KW, S, OH, OW, seg;   // conv geometry: seg = KW*Cin contiguous floats per kernel row
  FastDiv fd_per, fd_ow, fd_seg;       // OH*OW, OW, seg
  const float* bias;    // NN: [N] (or [1] when bias_shared)
  const float* bias2;   // NN dual: sigma bias [N]
  const float* a_scale; // NN dual: eps_in[K]; NT dual: eps_in[K] (output scale);  TN: eps_in[K]
  const float* c_scale; // NN dual: eps_out[N]; NT dual: eps_out[N]; TN: eps_out[N]
  const float* mul;     // NN: C = relu(..) * mul[(m / mul_div) * N + n]  (IQN Hadamard with the state embedding)
  const float* mask;    // NT: C *= (mask[m*ldc + k] > 0)   (ReLU backward)
  float* Cb;            // TN: bias-gradient row [N] (sum over m of G) or nullptr
  float* Cb2;           // TN: sigma-bias gradient [N] = c_scale * colsum(G)
  int mul_div;
  int relu;
  int bias_shared;
  int splits;           // split of the reduction dimension; partial s goes to C + s*split_stride (raw sums).
                        // NN: partial mode iff splits > 1;  TN: partial mode iff split_stride > 0
  long long split_stride;
};

constexpr int kMaxProblems = 6;
struct GemmBatch {
  GemmProblem p[kMaxProblems];
  int n;
};

// ---------------------------------------------------------------------------------------------
// A-operand addressing: element (m, k) of the (implicit) A matrix.
// ---------------------------------------------------------------------------------------------
struct ARow {
  const float* f;       // base of this row at k-segment 0 (nullptr if m out of range)
  const uint8_t* u;
};

__device__ __forceinline__ ARow a_row_base(const GemmProblem& p, int m) {
  ARow r{nullptr, nullptr};
  if (m >= p.M) return r;
  if (p.a_mode == A_PLAIN) {
    r.f = static_cast<const float*>(p.A) + (long long)m * p.lda;
  } else {
    int img = fd_div(m, p.fd_per), rem = m - img * p.fd_per.d;
    int oy = fd_div(rem, p.fd_ow), ox = rem - oy * p.fd_ow.d;
    long long off = ((long long)(oy * p.S) * p.W + ox * p.S) * p.Cin;
    if (p.a_mode == A_CONV_F32)
      r.f = static_cast<const float*>(p.A) + (long long)img * p.H * p.W * p.Cin + off;
    else
      r.u = static_cast<const uint8_t* const*>(p.A)[img] + off;
  }
  return r;
}

// x / 255 for an integer 0 <= x <= 255, correctly rounded: identical to __fdiv_rn(x, 255.f) for all 256
// inputs (checked exhaustively in tests/test_gpu_learner.py), without the IEEE division sequence.
__device__ __forceinline__ float u8_to_unit(unsigned int x) {
  const float inv = 0.0039215688593685627f;   // fl32(1/255)
  float xf = (float)x;
  float q = xf * inv;
  float r = fmaf(-q, 255.0f, xf);
  return fmaf(r, inv, q);
}

// Four consecutive k (k % 4 == 0) of row r: never straddles a kernel-row segment (seg % 4 == 0).
__device__ __forceinline__ float4 a_load4(const GemmProblem& p, const ARow& r, int k) {
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (k >= p.K) return v;
  if (p.a_mode == A_PLAIN) {
    if (r.f) v = *reinterpret_cast<const float4*>(r.f + k);
  } else {
    int kh = fd_div(k, p.fd_seg), rem = k - kh * p.fd_seg.d;
    int off = kh * p.W * p.Cin + rem;
    if (p.a_mode == A_CONV_F32) {
      if (r.f) v = *reinterpret_cast<const float4*>(r.f + off);
    } else if (r.u) {
      uchar4 b = *reinterpret_cast<const uchar4*>(r.u + off);
      v.x = u8_to_unit(b.x);   // x.astype(float32) / 255.0  (networks.py:193), correctly rounded
      v.y = u8_to_unit(b.y);
      v.z = u8_to_unit(b.z);
      v.w = u8_to_unit(b.w);
    }
  }
  return v;
}

template <int TM, int TN>
struct Acc {
  float v[TM][TN];
  __device__ __forceinline__ void clear() {
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
      for (int j = 0; j < TN; ++j) v[i][j] = 0.f;
  }
};

template <int N>
__device__ __forceinline__ void lds_vec(const float* p, float* out) {
  if constexpr (N == 8) {
    float4 t = *reinterpret_cast<const float4*>(p), u = *reinterpret_cast<const float4*>(p + 4);
    out[0] = t.x; out[1] = t.y; out[2] = t.z; out[3] = t.w; out[4] = u.x; out[5] = u.y; out[6] = u.z; out[7] = u.w;
  } else if constexpr (N == 4) {
    float4 t = *reinterpret_cast<const float4*>(p);
    out[0] = t.x; out[1] = t.y; out[2] = t.z; out[3] = t.w;
  } else if constexpr (N == 2) {
    float2 t = *reinterpret_cast<const float2*>(p);
    out[0] = t.x; out[1] = t.y;
  } else {
#pragma unroll
    for (int i = 0; i < N; ++i) out[i] = p[i];
  }
}

// One BK-deep rank update from shared tiles As[BK][BM+PAD], Bs[BK][BN+PAD] (vectorised LDS).
template <int BM, int BN, int BK, int TM, int TN, int PAD>
__device__ __forceinline__ void tile_fma(const float (*As)[BM + PAD], const float (*Bs)[BN + PAD], int ty, int tx,
                                         Acc<TM, TN>& acc) {
#pragma unroll
  for (int k = 0; k < BK; ++k) {
    float a[TM], b[TN];
    lds_vec<TM>(&As[k][ty * TM], a);
    lds_vec<TN>(&Bs[k][tx * TN], b);
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
      for (int j = 0; j < TN; ++j) acc.v[i][j] = fmaf(a[i], b[j], acc.v[i][j]);
  }
}

constexpr int kPad = 4;

__device__ __forceinline__ float4 ld4_guard(const float* src, int n, int N, bool vec) {
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (vec && n + 3 < N) return *reinterpret_cast<const float4*>(src);
  if (n + 0 < N) v.x = src[0];
  if (n + 1 < N) v.y = src[1];
  if (n + 2 < N) v.z = src[2];
  if (n + 3 < N) v.w = src[3];
  return v;
}

// All three kernels share one software pipeline: tiles are double buffered in shared memory and the
// next tile's global loads are issued into registers BEFORE the current tile's FMAs, so HBM/L2
// latency overlaps the math and there is one __syncthreads per k-step.

// ---------------------------------------------------------------------------------------------
// NN: C[M,N] = A[M,K] * B[K,N]  (+ dual accumulate for noisy layers, bias / ReLU / Hadamard epilogue)
// grid = (tiles_n, tiles_m * splits, problems)
// ---------------------------------------------------------------------------------------------
template <int BM, int BN, int BK, int TM, int TN, bool DUAL>
__global__ void __launch_bounds__((BM / TM) * (BN / TN)) gemm_nn_kernel(const __grid_constant__ GemmBatch batch) {
  dz::pdl_enter();
  constexpr int NT = (BM / TM) * (BN / TN);
  const GemmProblem& p = batch.p[blockIdx.z];
  const int tiles_m = (p.M + BM - 1) / BM;
  const int tile_m = blockIdx.y % tiles_m, split = blockIdx.y / tiles_m;
  const int m0 = tile_m * BM, n0 = blockIdx.x * BN;
  if (blockIdx.y >= tiles_m * p.splits || n0 >= p.N) return;
  const int kchunks = (p.K + BK - 1) / BK;
  const int per = (kchunks + p.splits - 1) / p.splits;
  const int kc0 = split * per, kc1 = min(kchunks, kc0 + per);

  __shared__ __align__(16) float As[2][BK][BM + kPad];
  __shared__ __align__(16) float Bs[2][BK][BN + kPad];

  const int tid = threadIdx.x, tx = tid % (BN / TN), ty = tid / (BN / TN);
  constexpr int A_VEC = BM * BK / 4, B_VEC = BK * BN / 4;
  constexpr int A_PER = (A_VEC + NT - 1) / NT, B_PER = (B_VEC + NT - 1) / NT;
  ARow rows[A_PER];
#pragma unroll
  for (int i = 0; i < A_PER; ++i) {
    int v = tid + i * NT;
    rows[i] = a_row_base(p, (v < A_VEC) ? m0 + v / (BK / 4) : p.M);
  }
  const bool vecB = (p.ldb % 4 == 0) && ((reinterpret_cast<uintptr_t>(p.B) & 15) == 0) &&
                    (!DUAL || (reinterpret_cast<uintptr_t>(p.B2) & 15) == 0);
  Acc<TM, TN> acc;
  acc.clear();

  // DUAL (noisy layers, networks.py:137-178): y = x Wmu + ((eps_in . x) Wsigma) . eps_out is evaluated as
  // x (Wmu + Wsigma . (eps_in (x) eps_out)): the effective weight tile is formed while the B tile is staged,
  // which halves the FMA work and the shared-memory traffic of these layers.
  float4 ra[A_PER], rb[B_PER];
  float4 eo[B_PER];                       // eps_out for this thread's 4 columns (fixed over k)
  if (DUAL) {
#pragma unroll
    for (int i = 0; i < B_PER; ++i) {
      int v = tid + i * NT;
      int nq = (v % (BN / 4)) * 4;
      eo[i] = (v < B_VEC) ? ld4_guard(p.c_scale + n0 + nq, n0 + nq, p.N, false) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  auto gload = [&](int kc) {
    const int k0 = kc * BK;
#pragma unroll
    for (int i = 0; i < A_PER; ++i) {
      int v = tid + i * NT;
      if (v < A_VEC) ra[i] = a_load4(p, rows[i], k0 + (v % (BK / 4)) * 4);
    }
#pragma unroll
    for (int i = 0; i < B_PER; ++i) {
      int v = tid + i * NT;
      if (v < B_VEC) {
        int kr = v / (BN / 4), nq = (v % (BN / 4)) * 4;
        int k = k0 + kr, n = n0 + nq;
        rb[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (k < p.K) {
          rb[i] = ld4_guard(p.B + (long long)k * p.ldb + n, n, p.N, vecB);
          if (DUAL) {
            float4 sg = ld4_guard(p.B2 + (long long)k * p.ldb + n, n, p.N, vecB);
            float ei = p.a_scale[k];
            rb[i].x = fmaf(sg.x, ei * eo[i].x, rb[i].x);
            rb[i].y = fmaf(sg.y, ei * eo[i].y, rb[i].y);
            rb[i].z = fmaf(sg.z, ei * eo[i].z, rb[i].z);
            rb[i].w = fmaf(sg.w, ei * eo[i].w, rb[i].w);
          }
        }
      }
    }
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int i = 0; i < A_PER; ++i) {
      int v = tid + i * NT;
      if (v < A_VEC) {
        int r = v / (BK / 4), kq = (v % (BK / 4)) * 4;
        float4 a = ra[i];
        As[buf][kq + 0][r] = a.x; As[buf][kq + 1][r] = a.y; As[buf][kq + 2][r] = a.z; As[buf][kq + 3][r] = a.w;
      }
    }
#pragma unroll
    for (int i = 0; i < B_PER; ++i) {
      int v = tid + i * NT;
      if (v < B_VEC) *reinterpret_cast<float4*>(&Bs[buf][v / (BN / 4)][(v % (BN / 4)) * 4]) = rb[i];
    }
  };

  if (kc0 < kc1) { gload(kc0); sstore(0); }
  __syncthreads();
  for (int kc = kc0; kc < kc1; ++kc) {
    const int cur = (kc - kc0) & 1;
    const bool more = kc + 1 < kc1;
    if (more) gload(kc + 1);
    tile_fma<BM, BN, BK, TM, TN, kPad>(As[cur], Bs[cur], ty, tx, acc);
    if (more) sstore(cur ^ 1);
    __syncthreads();
  }

  // epilogue
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    int m = m0 + ty * TM + i;
    if (m >= p.M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      int n = n0 + tx * TN + j;
      if (n >= p.N) continue;
      if (p.splits > 1) {
        p.C[(long long)split * p.split_stride + (long long)m * p.ldc + n] = acc.v[i][j];
        continue;
      }
      float v = acc.v[i][j];
      if (p.bias) v += p.bias_shared ? p.bias[0] : p.bias[n];
      if (DUAL && p.bias2) v = fmaf(p.bias2[n], p.c_scale[n], v);
      if (p.relu) v = fmaxf(v, 0.f);
      if (p.mul) {
        if (p.C2) p.C2[(long long)m * p.ldc + n] = v;
        v *= p.mul[(long long)(m / p.mul_div) * p.N + n];
      }
      p.C[(long long)m * p.ldc + n] = v;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// NN noisy layer with one noise apply per row (batched acting: actor stream m draws its own noise):
// C[m,n] = x[m,:] (Wmu + Wsigma . (eps_in[m] (x) eps_out[m]))[:,n], with row m's vectors at a_scale / c_scale +
// m * noise_ld.  Each mu / sigma tile is staged once per CTA for all BM rows and each row's weight is formed in
// registers with the operations and order of gemm_nn_kernel<DUAL> (t = eps_in * eps_out, w = fmaf(sigma, t, mu),
// acc = fmaf(x, w, acc)), over the same BK chunks, split boundaries and partial layout: rows that carry the same apply
// get that kernel's results bit for bit.  Plain A rows only.  grid = (tiles_n, tiles_m * splits, problems)
// ---------------------------------------------------------------------------------------------
template <int BM, int BN, int BK, int TM, int TN>
__global__ void __launch_bounds__((BM / TM) * (BN / TN))
    gemm_nn_rownoise_kernel(const __grid_constant__ GemmBatch batch, const long long noise_ld) {
  dz::pdl_enter();
  constexpr int NT = (BM / TM) * (BN / TN);
  const GemmProblem& p = batch.p[blockIdx.z];
  const int tiles_m = (p.M + BM - 1) / BM;
  const int tile_m = blockIdx.y % tiles_m, split = blockIdx.y / tiles_m;
  const int m0 = tile_m * BM, n0 = blockIdx.x * BN;
  if (blockIdx.y >= tiles_m * p.splits || n0 >= p.N) return;
  const int kchunks = (p.K + BK - 1) / BK;
  const int per = (kchunks + p.splits - 1) / p.splits;
  const int kc0 = split * per, kc1 = min(kchunks, kc0 + per);

  __shared__ __align__(16) float As[2][BK][BM + kPad];   // x
  __shared__ __align__(16) float Es[2][BK][BM + kPad];   // eps_in of each row
  __shared__ __align__(16) float Bs[2][BK][BN + kPad];   // mu
  __shared__ __align__(16) float Ss[2][BK][BN + kPad];   // sigma

  const int tid = threadIdx.x, tx = tid % (BN / TN), ty = tid / (BN / TN);
  constexpr int A_VEC = BM * BK / 4, B_VEC = BK * BN / 4;
  constexpr int A_PER = (A_VEC + NT - 1) / NT, B_PER = (B_VEC + NT - 1) / NT;
  ARow rows[A_PER];
  const float* ein[A_PER];
#pragma unroll
  for (int i = 0; i < A_PER; ++i) {
    int v = tid + i * NT;
    int m = (v < A_VEC) ? m0 + v / (BK / 4) : p.M;
    rows[i] = a_row_base(p, m);
    ein[i] = m < p.M ? p.a_scale + (long long)m * noise_ld : nullptr;
  }
  const bool vecB = (p.ldb % 4 == 0) && (((reinterpret_cast<uintptr_t>(p.B) | reinterpret_cast<uintptr_t>(p.B2)) & 15) == 0);
  const bool vecE = (noise_ld % 4 == 0) && ((reinterpret_cast<uintptr_t>(p.a_scale) & 15) == 0);
  float eo[TM][TN];   // eps_out of this thread's rows and columns (fixed over k)
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      int m = m0 + ty * TM + i, n = n0 + tx * TN + j;
      eo[i][j] = (m < p.M && n < p.N) ? p.c_scale[(long long)m * noise_ld + n] : 0.f;
    }
  Acc<TM, TN> acc;
  acc.clear();

  float4 ra[A_PER], re[A_PER], rb[B_PER], rs[B_PER];
  auto gload = [&](int kc) {
    const int k0 = kc * BK;
#pragma unroll
    for (int i = 0; i < A_PER; ++i) {
      int v = tid + i * NT;
      if (v < A_VEC) {
        int k = k0 + (v % (BK / 4)) * 4;
        ra[i] = a_load4(p, rows[i], k);
        re[i] = (ein[i] && k < p.K) ? ld4_guard(ein[i] + k, k, p.K, vecE) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
#pragma unroll
    for (int i = 0; i < B_PER; ++i) {
      int v = tid + i * NT;
      if (v < B_VEC) {
        int k = k0 + v / (BN / 4), n = n0 + (v % (BN / 4)) * 4;
        rb[i] = rs[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (k < p.K) {
          rb[i] = ld4_guard(p.B + (long long)k * p.ldb + n, n, p.N, vecB);
          rs[i] = ld4_guard(p.B2 + (long long)k * p.ldb + n, n, p.N, vecB);
        }
      }
    }
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int i = 0; i < A_PER; ++i) {
      int v = tid + i * NT;
      if (v < A_VEC) {
        int r = v / (BK / 4), kq = (v % (BK / 4)) * 4;
        As[buf][kq + 0][r] = ra[i].x; As[buf][kq + 1][r] = ra[i].y; As[buf][kq + 2][r] = ra[i].z; As[buf][kq + 3][r] = ra[i].w;
        Es[buf][kq + 0][r] = re[i].x; Es[buf][kq + 1][r] = re[i].y; Es[buf][kq + 2][r] = re[i].z; Es[buf][kq + 3][r] = re[i].w;
      }
    }
#pragma unroll
    for (int i = 0; i < B_PER; ++i) {
      int v = tid + i * NT;
      if (v < B_VEC) {
        *reinterpret_cast<float4*>(&Bs[buf][v / (BN / 4)][(v % (BN / 4)) * 4]) = rb[i];
        *reinterpret_cast<float4*>(&Ss[buf][v / (BN / 4)][(v % (BN / 4)) * 4]) = rs[i];
      }
    }
  };

  if (kc0 < kc1) { gload(kc0); sstore(0); }
  __syncthreads();
  for (int kc = kc0; kc < kc1; ++kc) {
    const int cur = (kc - kc0) & 1;
    const bool more = kc + 1 < kc1;
    if (more) gload(kc + 1);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[TM], e[TM], mu[TN], sg[TN];
      lds_vec<TM>(&As[cur][k][ty * TM], a);
      lds_vec<TM>(&Es[cur][k][ty * TM], e);
      lds_vec<TN>(&Bs[cur][k][tx * TN], mu);
      lds_vec<TN>(&Ss[cur][k][tx * TN], sg);
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) {
          const float w = fmaf(sg[j], e[i] * eo[i][j], mu[j]);
          acc.v[i][j] = fmaf(a[i], w, acc.v[i][j]);
        }
    }
    if (more) sstore(cur ^ 1);
    __syncthreads();
  }

  // epilogue (gemm_nn_kernel's, with row m's eps_out on the sigma bias)
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    int m = m0 + ty * TM + i;
    if (m >= p.M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      int n = n0 + tx * TN + j;
      if (n >= p.N) continue;
      if (p.splits > 1) {
        p.C[(long long)split * p.split_stride + (long long)m * p.ldc + n] = acc.v[i][j];
        continue;
      }
      float v = acc.v[i][j];
      if (p.bias) v += p.bias[n];
      if (p.bias2) v = fmaf(p.bias2[n], eo[i][j], v);
      if (p.relu) v = fmaxf(v, 0.f);
      p.C[(long long)m * p.ldc + n] = v;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// TN (weight gradient): C[K,N] = sum_m A[m,K]^T G[m,N].  Row K (one past the weights) accumulates
// the bias gradient (A treated as 1).  grid = (tiles_n, tiles_k * splits, problems); splits over m.
// ---------------------------------------------------------------------------------------------
template <int BMK, int BN, int BR, int TM, int TN>
__global__ void __launch_bounds__((BMK / TM) * (BN / TN)) gemm_tn_kernel(const __grid_constant__ GemmBatch batch) {
  dz::pdl_enter();
  constexpr int NT = (BMK / TM) * (BN / TN);
  const GemmProblem& p = batch.p[blockIdx.z];
  const int Kext = p.K + ((p.Cb || p.Cb2) ? 1 : 0);
  const int tiles_k = (Kext + BMK - 1) / BMK;
  const int tile_k = blockIdx.y % tiles_k, split = blockIdx.y / tiles_k;
  const int kk0 = tile_k * BMK, n0 = blockIdx.x * BN;
  if (blockIdx.y >= tiles_k * p.splits || n0 >= p.N) return;
  const int rchunks = (p.M + BR - 1) / BR;
  const int per = (rchunks + p.splits - 1) / p.splits;
  const int rc0 = split * per, rc1 = min(rchunks, rc0 + per);

  __shared__ __align__(16) float As[2][BR][BMK + kPad];
  __shared__ __align__(16) float Bs[2][BR][BN + kPad];
  const int tid = threadIdx.x, tx = tid % (BN / TN), ty = tid / (BN / TN);
  constexpr int A_VEC = BR * BMK / 4, B_VEC = BR * BN / 4;
  constexpr int A_PER = (A_VEC + NT - 1) / NT, B_PER = (B_VEC + NT - 1) / NT;
  const bool vecG = (p.ldb % 4 == 0) && ((reinterpret_cast<uintptr_t>(p.B) & 15) == 0);
  Acc<TM, TN> acc;
  acc.clear();
  float4 ra[A_PER], rb[B_PER];
  auto gload = [&](int rc) {
    const int r0 = rc * BR;
#pragma unroll
    for (int i = 0; i < A_PER; ++i) {
      int v = tid + i * NT;
      if (v < A_VEC) {
        int rr = v / (BMK / 4), kq = (v % (BMK / 4)) * 4;
        int m = r0 + rr, k = kk0 + kq;
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
        if (m < p.M) {
          if (k < p.K) {
            ARow row = a_row_base(p, m);
            a = a_load4(p, row, k);
          } else if (k == p.K) {
            a.x = 1.0f;  // bias-gradient row
          }
        }
        ra[i] = a;
      }
    }
#pragma unroll
    for (int i = 0; i < B_PER; ++i) {
      int v = tid + i * NT;
      if (v < B_VEC) {
        int rr = v / (BN / 4), nq = (v % (BN / 4)) * 4;
        int m = r0 + rr, n = n0 + nq;
        rb[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (m < p.M) rb[i] = ld4_guard(p.B + (long long)m * p.ldb + n, n, p.N, vecG);
      }
    }
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int i = 0; i < A_PER; ++i) {
      int v = tid + i * NT;
      if (v < A_VEC) *reinterpret_cast<float4*>(&As[buf][v / (BMK / 4)][(v % (BMK / 4)) * 4]) = ra[i];
    }
#pragma unroll
    for (int i = 0; i < B_PER; ++i) {
      int v = tid + i * NT;
      if (v < B_VEC) *reinterpret_cast<float4*>(&Bs[buf][v / (BN / 4)][(v % (BN / 4)) * 4]) = rb[i];
    }
  };
  if (rc0 < rc1) { gload(rc0); sstore(0); }
  __syncthreads();
  for (int rc = rc0; rc < rc1; ++rc) {
    const int cur = (rc - rc0) & 1;
    const bool more = rc + 1 < rc1;
    if (more) gload(rc + 1);
    tile_fma<BMK, BN, BR, TM, TN, kPad>(As[cur], Bs[cur], ty, tx, acc);
    if (more) sstore(cur ^ 1);
    __syncthreads();
  }

#pragma unroll
  for (int i = 0; i < TM; ++i) {
    int k = kk0 + ty * TM + i;
    if (k >= Kext) continue;
    const int nb = n0 + tx * TN;
    if (TN == 4 && nb + 3 < p.N && (p.N % 4 == 0) && (p.ldc % 4 == 0 || p.split_stride > 0)) {   // 16-byte stores
      float4 v4 = make_float4(acc.v[i][0], acc.v[i][1], acc.v[i][2], acc.v[i][3]);
      if (p.split_stride > 0) {
        *reinterpret_cast<float4*>(p.C + (long long)split * p.split_stride + (long long)k * p.N + nb) = v4;
        continue;
      }
      if (k < p.K) {
        if (p.C) *reinterpret_cast<float4*>(p.C + (long long)k * p.ldc + nb) = v4;
        if (p.C2) {
          float a = p.a_scale[k];
          float4 c = *reinterpret_cast<const float4*>(p.c_scale + nb);
          *reinterpret_cast<float4*>(p.C2 + (long long)k * p.ldc + nb) = make_float4(v4.x * a * c.x, v4.y * a * c.y, v4.z * a * c.z, v4.w * a * c.w);
        }
      } else {
        if (p.Cb) *reinterpret_cast<float4*>(p.Cb + nb) = v4;
        if (p.Cb2) {
          float4 c = *reinterpret_cast<const float4*>(p.c_scale + nb);
          *reinterpret_cast<float4*>(p.Cb2 + nb) = make_float4(v4.x * c.x, v4.y * c.y, v4.z * c.z, v4.w * c.w);
        }
      }
      continue;
    }
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      int n = n0 + tx * TN + j;
      if (n >= p.N) continue;
      float v = acc.v[i][j];
      if (p.split_stride > 0) {  // partial mode (even with a single split): raw sums, layout [Kext][N]
        p.C[(long long)split * p.split_stride + (long long)k * p.N + n] = v;
        continue;
      }
      if (k < p.K) {
        if (p.C) p.C[(long long)k * p.ldc + n] = v;
        if (p.C2) p.C2[(long long)k * p.ldc + n] = v * p.a_scale[k] * p.c_scale[n];
      } else {
        if (p.Cb) p.Cb[n] = v;
        if (p.Cb2) p.Cb2[n] = v * p.c_scale[n];
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// NT (input gradient): C[M,K] = G[M,N] * B[K,N]^T, optional dual (noisy) term and ReLU mask.
// grid = (tiles_k, tiles_m * splits, problems); splits over the reduction dim N: partial s (raw acc,
// then raw acc2 for DUAL) goes to C + s*split_stride with layout [M][K].
// ---------------------------------------------------------------------------------------------
template <int BM, int BNK, int BR, int TM, int TN, bool DUAL>
__global__ void __launch_bounds__((BM / TM) * (BNK / TN)) gemm_nt_kernel(const __grid_constant__ GemmBatch batch) {
  dz::pdl_enter();
  constexpr int NT = (BM / TM) * (BNK / TN);
  const GemmProblem& p = batch.p[blockIdx.z];
  const int tiles_m = (p.M + BM - 1) / BM;
  const int tile_m = blockIdx.y % tiles_m, split = blockIdx.y / tiles_m;
  const int m0 = tile_m * BM, k0 = blockIdx.x * BNK;
  if (blockIdx.y >= tiles_m * p.splits || k0 >= p.K) return;
  const int nchunks = (p.N + BR - 1) / BR;
  const int per = (nchunks + p.splits - 1) / p.splits;
  const int nc0 = split * per, nc1 = min(nchunks, nc0 + per);
  __shared__ __align__(16) float As[2][BR][BM + kPad];
  __shared__ __align__(16) float Bs[2][BR][BNK + kPad];
  const int tid = threadIdx.x, tx = tid % (BNK / TN), ty = tid / (BNK / TN);
  const bool vec = (p.ldb % 4 == 0) && ((reinterpret_cast<uintptr_t>(p.B) & 15) == 0) &&
                   ((reinterpret_cast<uintptr_t>(p.A) & 15) == 0) && (p.lda % 4 == 0) &&
                   (!DUAL || (reinterpret_cast<uintptr_t>(p.B2) & 15) == 0);
  const float* G = static_cast<const float*>(p.A);
  Acc<TM, TN> acc;
  acc.clear();
  constexpr int A_VEC = BM * BR / 4, B_VEC = BNK * BR / 4;
  constexpr int A_PER = (A_VEC + NT - 1) / NT, B_PER = (B_VEC + NT - 1) / NT;
  float4 ra[A_PER], rb[B_PER];
  // DUAL: dx = g (Wmu + Wsigma . (eps_in (x) eps_out))^T — effective weights formed while staging the B tile.
  auto gload = [&](int nc) {
    const int n0 = nc * BR;
#pragma unroll
    for (int i = 0; i < A_PER; ++i) {
      int v = tid + i * NT;
      if (v < A_VEC) {
        int r = v / (BR / 4), nq = (v % (BR / 4)) * 4;
        int m = m0 + r, n = n0 + nq;
        ra[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (m < p.M) ra[i] = ld4_guard(G + (long long)m * p.lda + n, n, p.N, vec);
      }
    }
#pragma unroll
    for (int i = 0; i < B_PER; ++i) {
      int v = tid + i * NT;
      if (v < B_VEC) {
        int kr = v / (BR / 4), nq = (v % (BR / 4)) * 4;
        int k = k0 + kr, n = n0 + nq;
        rb[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (k < p.K) {
          rb[i] = ld4_guard(p.B + (long long)k * p.ldb + n, n, p.N, vec);
          if (DUAL) {
            float4 sg = ld4_guard(p.B2 + (long long)k * p.ldb + n, n, p.N, vec);
            float4 eo = ld4_guard(p.c_scale + n, n, p.N, false);
            float ei = p.a_scale[k];
            rb[i].x = fmaf(sg.x, ei * eo.x, rb[i].x);
            rb[i].y = fmaf(sg.y, ei * eo.y, rb[i].y);
            rb[i].z = fmaf(sg.z, ei * eo.z, rb[i].z);
            rb[i].w = fmaf(sg.w, ei * eo.w, rb[i].w);
          }
        }
      }
    }
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int i = 0; i < A_PER; ++i) {
      int v = tid + i * NT;
      if (v < A_VEC) {
        int r = v / (BR / 4), nq = (v % (BR / 4)) * 4;
        float4 g = ra[i];
        As[buf][nq + 0][r] = g.x; As[buf][nq + 1][r] = g.y; As[buf][nq + 2][r] = g.z; As[buf][nq + 3][r] = g.w;
      }
    }
#pragma unroll
    for (int i = 0; i < B_PER; ++i) {
      int v = tid + i * NT;
      if (v < B_VEC) {
        int kr = v / (BR / 4), nq = (v % (BR / 4)) * 4;
        float4 b = rb[i];
        Bs[buf][nq + 0][kr] = b.x; Bs[buf][nq + 1][kr] = b.y; Bs[buf][nq + 2][kr] = b.z; Bs[buf][nq + 3][kr] = b.w;
      }
    }
  };
  if (nc0 < nc1) { gload(nc0); sstore(0); }
  __syncthreads();
  for (int nc = nc0; nc < nc1; ++nc) {
    const int cur = (nc - nc0) & 1;
    const bool more = nc + 1 < nc1;
    if (more) gload(nc + 1);
    tile_fma<BM, BNK, BR, TM, TN, kPad>(As[cur], Bs[cur], ty, tx, acc);
    if (more) sstore(cur ^ 1);
    __syncthreads();
  }

#pragma unroll
  for (int i = 0; i < TM; ++i) {
    int m = m0 + ty * TM + i;
    if (m >= p.M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      int k = k0 + tx * TN + j;
      if (k >= p.K) continue;
      if (p.splits > 1) {
        p.C[(long long)split * p.split_stride + (long long)m * p.K + k] = acc.v[i][j];
        continue;
      }
      float v = acc.v[i][j];
      if (p.mask && !(p.mask[(long long)m * p.ldc + k] > 0.f)) v = 0.f;
      p.C[(long long)m * p.ldc + k] = v;
    }
  }
}

}  // namespace dz
