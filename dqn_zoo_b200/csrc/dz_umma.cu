// Host side of the TMA-fed tensor-core GEMM family + a C-ABI self test (plain GEMMs through every operand path).
#include <cudaTypedefs.h>

#include "dz_umma_host.cuh"

namespace dz {

namespace {

PFN_cuTensorMapEncodeTiled_v12000 encode_fn() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  }
  return fn;
}

}  // namespace

int UmPlan::add_map(const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box) {
  auto fn = encode_fn();
  if (!fn) { fail(DZ_ECUDA, "cuTensorMapEncodeTiled entry point not available"); return -1; }
  cuuint64_t gd[5] = {1, 1, 1, 1, 1};
  cuuint64_t gs[4] = {16, 16, 16, 16};
  cuuint32_t bx[5] = {1, 1, 1, 1, 1};
  cuuint32_t es[5] = {1, 1, 1, 1, 1};
  uint64_t last = 16;
  for (int i = 0; i < 5; ++i) {
    if (i < rank) { gd[i] = dims[i]; bx[i] = box[i]; }
    if (i >= 1) {
      if (i < rank) gs[i - 1] = strides_bytes[i - 1];
      else gs[i - 1] = last;                  // size-1 dimension: any legal stride
      last = gs[i - 1] * gd[i];
      if (last % 16) last = (last + 15) / 16 * 16;
    } else {
      last = gd[0] * 4;
      if (last % 16) last = (last + 15) / 16 * 16;
    }
  }
  if (bx[0] * 4 > 128) { fail(DZ_EINVAL, "tensor map: inner box wider than the 128-byte swizzle span"); return -1; }
  CUtensorMap m;
  CUresult rc = fn(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, const_cast<void*>(base), gd, gs, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (rc != CUDA_SUCCESS) {
    char buf[256];
    snprintf(buf, sizeof(buf), "cuTensorMapEncodeTiled failed (%d): dims %llu %llu %llu %llu %llu strides %llu %llu %llu %llu box %u %u %u %u %u", (int)rc,
             (unsigned long long)gd[0], (unsigned long long)gd[1], (unsigned long long)gd[2], (unsigned long long)gd[3], (unsigned long long)gd[4],
             (unsigned long long)gs[0], (unsigned long long)gs[1], (unsigned long long)gs[2], (unsigned long long)gs[3], bx[0], bx[1], bx[2], bx[3], bx[4]);
    g_last_error = buf;
    return -1;
  }
  maps.push_back(m);
  box_bytes.push_back(bx[0] * bx[1] * bx[2] * bx[3] * bx[4] * 4);
  return (int)maps.size() - 1;
}

int UmPlan::add_map_pair(const float* hi, const float* lo, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                         const uint32_t* box, int ids[2]) {
  ids[0] = add_map(hi, rank, dims, strides_bytes, box);
  ids[1] = ids[0] < 0 ? -1 : add_map(lo, rank, dims, strides_bytes, box);
  return ids[1] < 0 ? DZ_EINVAL : DZ_OK;
}

int UmPlan::end_cta() {
  UmCta& c = ctas.back();
  const size_t nst = stage_op0.size();
  c.nstages = (uint32_t)nst;
  for (size_t s = 0; s < nst; ++s) {
    const uint32_t o1 = s + 1 < nst ? stage_op0[s + 1] : (uint32_t)ops.size();
    uint32_t tx = 0;
    for (uint32_t oi = stage_op0[s]; oi < o1; ++oi) {
      const uint32_t bytes = box_bytes[ops[oi].map];
      if (ops[oi].smem_off + bytes > build_stage_bytes) return fail(DZ_EINVAL, "umma plan: a TMA box overruns its stage");
      tx += bytes;
    }
    const uint32_t nops = o1 - stage_op0[s];
    if (nops > 32) return fail(DZ_EINVAL, "umma plan: more than 32 TMA ops in one stage");
    if (s == 0) { c.ops_per_stage = nops; c.tx_bytes = tx; }
    else if (nops != c.ops_per_stage || tx != c.tx_bytes) return fail(DZ_EINVAL, "umma plan: the stages of a CTA differ in TMA ops or bytes");
  }
  return DZ_OK;
}

int UmPlan::localize_maps(UmLaunch& l) {
  l.nmaps = 0;
  for (int ci = l.cta0; ci < l.cta0 + l.nctas; ++ci) {
    const UmCta& c = ctas[ci];
    const size_t n = (size_t)c.nstages * c.ops_per_stage;
    for (size_t oi = c.op0; oi < c.op0 + n; ++oi) {
      const int id = (int)ops[oi].map;
      int slot = -1;
      for (int q = 0; q < l.nmaps; ++q) if (l.map_ids[q] == id) slot = q;
      if (slot < 0) {
        if (l.nmaps >= um::kMaxMapsPerLaunch) return fail(DZ_EINVAL, "too many tensor maps in one launch");
        slot = l.nmaps;
        l.map_ids[l.nmaps++] = id;
      }
      ops[oi].map = (uint32_t)slot;
    }
  }
  return DZ_OK;
}

void UmPlan::release() {
  if (d_maps) cudaFree(d_maps);
  if (d_probs) cudaFree(d_probs);
  if (d_ctas) cudaFree(d_ctas);
  if (d_ops) cudaFree(d_ops);
  d_maps = nullptr; d_probs = nullptr; d_ctas = nullptr; d_ops = nullptr;
}

int UmPlan::upload() {
  release();
  if (maps.empty() || probs.empty() || ctas.empty() || ops.empty()) return fail(DZ_EINVAL, "empty umma plan");
  DZ_CUDA_OK(cudaMalloc(&d_maps, maps.size() * sizeof(CUtensorMap)));
  DZ_CUDA_OK(cudaMalloc(&d_probs, probs.size() * sizeof(UmProblem)));
  DZ_CUDA_OK(cudaMalloc(&d_ctas, ctas.size() * sizeof(UmCta)));
  DZ_CUDA_OK(cudaMalloc(&d_ops, ops.size() * sizeof(UmTmaOp)));
  DZ_CUDA_OK(cudaMemcpy(d_maps, maps.data(), maps.size() * sizeof(CUtensorMap), cudaMemcpyHostToDevice));
  DZ_CUDA_OK(cudaMemcpy(d_probs, probs.data(), probs.size() * sizeof(UmProblem), cudaMemcpyHostToDevice));
  DZ_CUDA_OK(cudaMemcpy(d_ctas, ctas.data(), ctas.size() * sizeof(UmCta), cudaMemcpyHostToDevice));
  DZ_CUDA_OK(cudaMemcpy(d_ops, ops.data(), ops.size() * sizeof(UmTmaOp), cudaMemcpyHostToDevice));
  return DZ_OK;
}

int UmPlan::configure() {
  static bool done = false;
  if (done) return DZ_OK;
  DZ_CUDA_OK(cudaFuncSetAttribute(um::umma_gemm_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  DZ_CUDA_OK(cudaFuncSetAttribute(um::umma_gemm_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  DZ_CUDA_OK(cudaFuncSetAttribute(um::umma_fc_kernel<32, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  DZ_CUDA_OK(cudaFuncSetAttribute(um::umma_fc_kernel<64, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  DZ_CUDA_OK(cudaFuncSetAttribute(um::umma_fc_kernel<32, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  DZ_CUDA_OK(cudaFuncSetAttribute(um::umma_fc_kernel<64, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  DZ_CUDA_OK(cudaFuncSetAttribute(um::wgmma_gemm_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  DZ_CUDA_OK(cudaFuncSetAttribute(um::wgmma_gemm_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  done = true;
  return DZ_OK;
}

bool UmPlan::wgmma_eligible(const UmLaunch& l) const {
  for (int ci = l.cta0; ci < l.cta0 + l.nctas; ++ci) {
    const UmProblem& pr = probs[ctas[ci].prob];
    for (const UmOperand* o : {&pr.A, &pr.B})
      if (o->mn_major || o->nparts != 2 || o->convert) return false;
    if (pr.ksteps != 4) return false;
  }
  return true;
}

bool UmPlan::fc_eligible(const UmLaunch& l) const {
  for (int ci = l.cta0; ci < l.cta0 + l.nctas; ++ci) {
    const UmCta& c = ctas[ci];
    const int np = c.nprob > 1 ? (int)c.nprob : 1;
    if (np > um::kFcMaxProbs) return false;
    for (int q = 0; q < np; ++q) {
      const UmProblem& pr = probs[c.prob + q];
      if (pr.A.mn_major != probs[ctas[l.cta0].prob].A.mn_major) return false;   // one A layout per launch
      if (pr.A.mn_major ? pr.A.lbo != 4096u : np != 1) return false;
      if (pr.A.part_bytes * (uint32_t)np != 16384u) return false;
      if (pr.A.convert != 2 && !(pr.A.convert == 1 && pr.A.scale_r == nullptr)) return false;
      if (pr.B.mn_major || pr.B.nparts != 2 || pr.B.convert) return false;
      if (pr.ksteps != 4 || pr.red_per_stage != 32 || pr.epi != UM_EPI_PARTIAL || pr.sc_i != 1) return false;
      if (q > 0 && (pr.A.part_bytes != probs[c.prob].A.part_bytes || pr.A.convert != probs[c.prob].A.convert ||
                    pr.B.part_bytes != probs[c.prob].B.part_bytes))
        return false;
    }
    if (2 * 16384u / (uint32_t)np + (uint32_t)np * 2u * probs[c.prob].B.part_bytes > l.stage_bytes) return false;
  }
  return true;
}

int UmPlan::launch(const char* tag, const UmLaunch& l, void* stream, long long* d_trace, int path) const {
  if (l.nctas <= 0) return DZ_OK;
  if (!d_ctas) return fail(DZ_EINVAL, "umma plan not uploaded");
  if (l.stages < 1 || l.stages > um::kStagesMax || l.stage_bytes % 1024) return fail(DZ_EINVAL, "umma launch geometry");
  for (int ci = l.cta0; ci < l.cta0 + l.nctas; ++ci) {
    const UmProblem& pr = probs[ctas[ci].prob];
    const uint32_t want = pr.B.mn_major ? (uint32_t)(l.njt / 32) * pr.B.lbo : (uint32_t)l.njt * 128u;
    if (pr.A.nparts != 2 || pr.B.nparts != 2 || pr.B.part_bytes != want)
      return fail(DZ_EINVAL, "umma launch: operands must be hi/lo pairs and the B tile must span NJT rows");
  }
  const int stages = l.stages;
  const size_t smem = um_smem_bytes(stages, l.stage_bytes);
  if (smem > 227 * 1024) return fail(DZ_EINVAL, "umma launch needs too much shared memory");
  if ((size_t)stages * l.stage_bytes < (size_t)128 * l.njt * 4) return fail(DZ_EINVAL, "umma launch: stage buffers smaller than the store-phase staging tile");
  const int v = l.njt == 32 ? 0 : 1;
  if (l.njt != 32 && l.njt != 64) return fail(DZ_EINVAL, "umma launch: NJT must be 32 or 64");
  if (path != UM_PATH_AUTO && path != UM_PATH_MMA_SYNC && path != UM_PATH_WGMMA && path != UM_PATH_CONVERTERS)
    return fail(DZ_EINVAL, "umma launch: unknown MMA path");
  const bool wg = path == UM_PATH_AUTO ? wgmma_eligible(l) : path == UM_PATH_WGMMA;
  if (wg && !wgmma_eligible(l)) return fail(DZ_EINVAL, "umma launch: the wgmma path needs K-major, pre-split operands and four k-steps per stage");
  if (wg)
    for (int ci = l.cta0; ci < l.cta0 + l.nctas; ++ci)
      if (um_wgmma_min_stage(probs[ctas[ci].prob].A.part_bytes) > l.stage_bytes) return fail(DZ_EINVAL, "umma launch: stage too small for the wgmma A reads");
  DZ_TRY(configure());
  um::UmMaps lm;
  for (int q = 0; q < l.nmaps; ++q) lm.m[q] = maps[l.map_ids[q]];
  for (int q = l.nmaps; q < um::kMaxMapsPerLaunch; ++q) lm.m[q] = maps[l.map_ids[0]];
  if (wg) {
    if (v == 0)
      DZ_LAUNCH_NAMED(tag, um::wgmma_gemm_kernel<32>, (unsigned)l.nctas, um::kThreadsW, smem, stream, lm, d_ctas + l.cta0, d_probs, d_ops, l.nmaps,
                      stages, l.stage_bytes, d_trace);
    else
      DZ_LAUNCH_NAMED(tag, um::wgmma_gemm_kernel<64>, (unsigned)l.nctas, um::kThreadsW, smem, stream, lm, d_ctas + l.cta0, d_probs, d_ops, l.nmaps,
                      stages, l.stage_bytes, d_trace);
    return DZ_OK;
  }
  if (path != UM_PATH_CONVERTERS && fc_eligible(l)) {
    const bool ak = !probs[ctas[l.cta0].prob].A.mn_major;
    auto kern = v == 0 ? (ak ? um::umma_fc_kernel<32, true> : um::umma_fc_kernel<32, false>)
                       : (ak ? um::umma_fc_kernel<64, true> : um::umma_fc_kernel<64, false>);
    DZ_LAUNCH_NAMED(tag, kern, (unsigned)l.nctas, um::kThreadsF, smem, stream, lm, d_ctas + l.cta0, d_probs, d_ops, l.nmaps, stages,
                    l.stage_bytes, d_trace);
    return DZ_OK;
  }
  for (int ci = l.cta0; ci < l.cta0 + l.nctas; ++ci)
    if (ctas[ci].nprob > 1) return fail(DZ_EINVAL, "umma launch: CTAs that serve several problems need umma_fc_kernel");
  if (v == 0)
    DZ_LAUNCH_NAMED(tag, um::umma_gemm_kernel<32>, (unsigned)l.nctas, um::kThreadsU, smem, stream, lm, d_ctas + l.cta0, d_probs, d_ops, l.nmaps, stages,
                    l.stage_bytes, d_trace);
  else
    DZ_LAUNCH_NAMED(tag, um::umma_gemm_kernel<64>, (unsigned)l.nctas, um::kThreadsU, smem, stream, lm, d_ctas + l.cta0, d_probs, d_ops, l.nmaps, stages,
                    l.stage_bytes, d_trace);
  return DZ_OK;
}

namespace {
__global__ void um_split_kernel(const float* __restrict__ x, float* __restrict__ hi, float* __restrict__ lo, long long n) {
  dz::pdl_enter();
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < n) {
    float h, l;
    tc::split_tf32(x[i], h, l);
    hi[i] = h;
    lo[i] = l;
  }
}
}  // namespace

int um_split(const float* x, float* hi, float* lo, long long n, void* stream) {
  DZ_LAUNCH(um_split_kernel, (unsigned)ceil_div(n, 256), 256, 0, stream, x, hi, lo, n);
  return DZ_OK;
}

}  // namespace dz

using namespace dz;

// Self test: C[MI][NJ] = sum_r A(i,r) B(j,r); NJ and R multiples of 4, and MI too when A is MN-major (TMA row strides).
//   a_mn_major = 0: d_A is [MI][R] (K-major source);  1: d_A is [R][MI] (MN-major source).  Same for B with NJ <= 64.
//   convert = 0: operands are split into hi/lo by a helper kernel first (the layout the activations use);
//   convert = 1: raw fp32 tiles are split in shared memory by the converter warps (the layout the weights use),
//                optionally scaled by d_scale_r[r] (applied to A).
//   epi_rows = 1: UM_EPI_ROWS epilogue (+ d_bias[j], relu, tf32 hi/lo outputs in d_hi / d_lo besides d_C).
//   path: 0 automatic (as the learner's launches), 1 mma.sync kernel, 2 wgmma kernel (K-major pre-split operands only).
extern "C" int dz_test_umma_gemm_path(const float* d_A, int32_t a_mn_major, const float* d_B, int32_t b_mn_major, int32_t MI,
                                      int32_t NJ, int32_t R, int32_t convert, const float* d_scale_r, int32_t stages,
                                      int32_t epi_rows, const float* d_bias, int32_t relu, float* d_C, float* d_hi, float* d_lo,
                                      int32_t path, void* stream) {
  if (NJ < 4 || NJ > 64 || NJ % 4 || (a_mn_major && MI % 4) || R % 4) return fail(DZ_EINVAL, "umma self test extents");
  const int njt = NJ <= 32 ? 32 : 64;
  UmPlan plan;
  float *a_hi = nullptr, *a_lo = nullptr, *b_hi = nullptr, *b_lo = nullptr;
  const long long na = (long long)MI * R, nb = (long long)NJ * R;
  if (!convert) {
    DZ_CUDA_OK(cudaMalloc(&a_hi, na * 4)); DZ_CUDA_OK(cudaMalloc(&a_lo, na * 4));
    DZ_CUDA_OK(cudaMalloc(&b_hi, nb * 4)); DZ_CUDA_OK(cudaMalloc(&b_lo, nb * 4));
    int rc = um_split(d_A, a_hi, a_lo, na, stream);
    if (rc == DZ_OK) rc = um_split(d_B, b_hi, b_lo, nb, stream);
    if (rc != DZ_OK) return rc;
  }
  const int nparts = convert ? 1 : 2;   // convert: one raw fp32 map per operand
  auto make_maps = [&](const float* hi, const float* lo, int mn_major, int rows, int tile_rows, int out[2]) -> int {
    uint64_t dims[2], strides[1];
    uint32_t box[2];
    if (!mn_major) { dims[0] = (uint64_t)R; dims[1] = (uint64_t)rows; strides[0] = (uint64_t)R * 4; box[0] = 32; box[1] = (uint32_t)tile_rows; }
    else { dims[0] = (uint64_t)rows; dims[1] = (uint64_t)R; strides[0] = (uint64_t)rows * 4; box[0] = 32; box[1] = 32; }
    if (nparts == 2) return plan.add_map_pair(hi, lo, 2, dims, strides, box, out);
    out[0] = plan.add_map(hi, 2, dims, strides, box);
    return out[0] < 0 ? DZ_EINVAL : DZ_OK;
  };
  int ma[2] = {-1, -1}, mb[2] = {-1, -1};
  int rc = make_maps(convert ? d_A : a_hi, a_lo, a_mn_major, MI, 128, ma);
  if (rc == DZ_OK) rc = make_maps(convert ? d_B : b_hi, b_lo, b_mn_major, NJ, njt, mb);
  if (rc != DZ_OK) return rc;

  UmProblem p;
  memset(&p, 0, sizeof(p));
  p.A = a_mn_major ? um_mnmajor(128, 32, convert != 0, convert ? d_scale_r : nullptr) : um_kmajor(128, true, convert != 0, convert ? d_scale_r : nullptr);
  p.B = b_mn_major ? um_mnmajor(njt, 32, convert != 0) : um_kmajor(njt, true, convert != 0);
  p.ksteps = 4; p.red_per_stage = 32;
  p.MI = MI; p.NJ = NJ;
  if (epi_rows) {
    p.epi = UM_EPI_ROWS; p.out_f32 = d_C; p.out_hi = d_hi; p.out_lo = d_lo; p.bias = d_bias; p.relu = relu;
    p.pw = 1 << 20; p.rs_outer = 0; p.rs_inner = 1; p.out_ld = NJ;
  } else {
    p.epi = UM_EPI_PARTIAL; p.C = d_C; p.sc_i = NJ; p.sc_j = 1; p.split_stride = 0;
  }
  const int prob = plan.add_problem(p);
  const int nst = (int)ceil_div(R, 32);
  const uint32_t a_bytes = p.A.part_bytes * 2, b_bytes = p.B.part_bytes * 2;
  const int tiles = (int)ceil_div(MI, 128);
  UmLaunch l;
  plan.begin_launch(l, njt, a_bytes + b_bytes);
  l.stages = stages > 0 ? stages : 4;   // 4 x <= 48 KB + control block fits
  for (int t = 0; t < tiles && rc == DZ_OK; ++t) {
    UmCta& c = plan.begin_cta(prob);
    c.i0 = t * 128; c.row_base = t * 128; c.ph_valid = 1; c.pw_valid = std::min(128, MI - t * 128);
    for (int s = 0; s < nst; ++s) {
      plan.stage();
      for (int part = 0; part < nparts; ++part) {
        const uint32_t base = part * p.A.part_bytes;
        if (!a_mn_major) plan.op(ma[part], base, 32 * s, t * 128);
        else for (int q = 0; q < 4; ++q) plan.op(ma[part], base + q * 4096, t * 128 + 32 * q, 32 * s);
      }
      for (int part = 0; part < nparts; ++part) {
        const uint32_t base = a_bytes + part * p.B.part_bytes;
        if (!b_mn_major) plan.op(mb[part], base, 32 * s, 0);
        else for (int q = 0; q < njt / 32; ++q) plan.op(mb[part], base + q * 4096, 32 * q, 32 * s);
      }
    }
    rc = plan.end_cta();
  }
  plan.end_launch(l);
  if (rc == DZ_OK) rc = plan.localize_maps(l);
  if (rc == DZ_OK) rc = plan.upload();
  if (rc != DZ_OK) return rc;
  rc = plan.launch("umma_selftest", l, stream, nullptr, path);
  cudaError_t e = cudaStreamSynchronize((cudaStream_t)stream);
  plan.release();
  if (a_hi) { cudaFree(a_hi); cudaFree(a_lo); cudaFree(b_hi); cudaFree(b_lo); }
  if (rc != DZ_OK) return rc;
  if (e != cudaSuccess) return fail(DZ_ECUDA, "umma self test: %s", cudaGetErrorString(e));
  return DZ_OK;
}

extern "C" int dz_test_umma_gemm(const float* d_A, int32_t a_mn_major, const float* d_B, int32_t b_mn_major, int32_t MI, int32_t NJ,
                                 int32_t R, int32_t convert, const float* d_scale_r, int32_t stages, int32_t epi_rows,
                                 const float* d_bias, int32_t relu, float* d_C, float* d_hi, float* d_lo, void* stream) {
  return dz_test_umma_gemm_path(d_A, a_mn_major, d_B, b_mn_major, MI, NJ, R, convert, d_scale_r, stages, epi_rows, d_bias, relu,
                                d_C, d_hi, d_lo, UM_PATH_AUTO, stream);
}
