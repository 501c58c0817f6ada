// Host-side launchers of the packed-operand tensor-core GEMM (dz_tcp.cuh) + a C-ABI self-test entry point.
#include "dz_tcp.cuh"
#include "dz_internal.cuh"

namespace dz {

int pk_add_job(PackBatch& pb, const float* src, int ld, int red_contig, int rows, int red, int rows_pad, int red_pad,
               int ones_row, float* hi, float* lo) {
  if (pb.n >= kPkMaxJobs) return fail(DZ_EINVAL, "too many pack jobs");
  if (rows_pad % 128 || red_pad % kPkKB || rows_pad < rows || red_pad < red || (ones_row >= rows_pad))
    return fail(DZ_EINVAL, "pack job extents");
  PackJob& j = pb.job[pb.n++];
  j.src = src; j.ld = ld; j.red_contig = red_contig; j.rows = rows; j.red = red; j.rows_pad = rows_pad; j.red_pad = red_pad;
  j.ones_row = ones_row; j.hi = hi; j.lo = lo;
  j.tiles_r = ceil_div(rows_pad, 64);
  j.block0 = pb.blocks;
  pb.blocks += j.tiles_r * (int)ceil_div(red_pad, 64);
  return DZ_OK;
}

namespace {
__global__ void pk_ones_row_kernel(float* hi, int rg_total, int row, int red) {
  dz::pdl_enter();
  int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m < red) hi[pk_index(row, m, rg_total)] = 1.f;
}
}  // namespace

int pk_set_ones_row(float* hi, int rows_pad, int row, int red, void* stream) {
  DZ_LAUNCH(pk_ones_row_kernel, (unsigned)ceil_div(red, 256), 256, 0, stream, hi, rows_pad / 8, row, red);
  return DZ_OK;
}

int launch_pack(const char* tag, const PackBatch& pb, void* stream) {
  if (pb.n <= 0) return DZ_OK;
  DZ_LAUNCH_NAMED(tag, tcp::tc_pack_kernel, (unsigned)pb.blocks, 256, 0, stream, pb);
  return DZ_OK;
}

template <int EPI>
static int launch_pgemm_t(const char* tag, const PkBatch& kb, void* stream) {
  constexpr int BNJ = 256;
  using L = tcp::PkSmem<BNJ, EPI>;
  static bool configured = false;
  if (!configured) {
    DZ_CUDA_OK(cudaFuncSetAttribute(tcp::tc_pgemm_kernel<BNJ, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::kTotal));
    configured = true;
  }
  int max_i = 0, max_j = 0, max_s = 1;
  for (int q = 0; q < kb.n; ++q) {
    const PkProblem& p = kb.p[q];
    if (p.splits < 1 || p.nkb < 1) return fail(DZ_EINVAL, "pgemm problem");
    if (p.A.rg_total * 8 < ceil_div(p.MI, 128) * 128 || p.B.rg_total * 8 < ceil_div(p.NJ, BNJ) * BNJ)
      return fail(DZ_EINVAL, "pgemm operand images are not padded to the tile size");
    if (EPI == 1 && (p.splits != 1 || p.nkb > 8 || p.NJ % 4 || p.MI % 4 || !p.bias_j || !p.mul || !p.img_hi || p.mul_div < 1))
      return fail(DZ_EINVAL, "pgemm embedding epilogue arguments");
    max_i = p.MI > max_i ? p.MI : max_i;
    max_j = p.NJ > max_j ? p.NJ : max_j;
    max_s = p.splits > max_s ? p.splits : max_s;
  }
  dim3 grid((unsigned)ceil_div(max_j, BNJ), (unsigned)(ceil_div(max_i, 128) * max_s), kb.n);
  DZ_LAUNCH_NAMED(tag, (tcp::tc_pgemm_kernel<BNJ, EPI>), grid, tcp::kThreadsP, L::kTotal, stream, kb);
  return DZ_OK;
}

int launch_pgemm(const char* tag, const PkBatch& kb, void* stream, int epi) {
  if (kb.n <= 0 || kb.n > kPkMaxProblems) return fail(DZ_EINVAL, "pgemm batch size");
  return epi ? launch_pgemm_t<1>(tag, kb, stream) : launch_pgemm_t<0>(tag, kb, stream);
}

PkProblem pk_embed_problem(const PkOperand& cos, const PkOperand& weT, int M, int D, int nkb, const float* bias,
                           const float* mul, int mul_div, int mul_ld, float* e0, const PkTarget& img, const PkTarget& imgT) {
  PkProblem p;
  memset(&p, 0, sizeof(p));
  p.A = cos; p.B = weT;
  p.MI = M; p.NJ = D; p.nkb = nkb; p.splits = 1;
  p.bias_j = bias;
  p.mul = mul; p.mul_div = mul_div; p.mul_ld = mul_ld;
  p.e0 = e0; p.e0_ld = D;
  p.img_hi = img.hi; p.img_lo = img.lo; p.img_rg = img.rg;
  if (imgT.hi) { p.imgT_hi = imgT.hi; p.imgT_lo = imgT.lo; p.imgT_rg = imgT.rg; }
  return p;
}

}  // namespace dz

using namespace dz;

// Self test: D[i,j] = sum_r A(i,r) B(j,r) with both operands packed from plain fp32 matrices in either
// orientation.  d_work must hold 2 * (a_rows_pad + b_rows_pad) * red_pad floats (see dz_test_tc_pgemm_work).
extern "C" int64_t dz_test_tc_pgemm_work(int32_t a_rows, int32_t b_rows, int32_t red) {
  int64_t ar = ceil_div(a_rows + 1, 128) * 128, br = ceil_div(b_rows, 256) * 256, rp = ceil_div(red, kPkKB) * kPkKB;
  return 2 * (ar + br) * rp;
}

extern "C" int dz_test_tc_pgemm(const float* d_A, int32_t a_rows, int32_t a_ld, int32_t a_red_contig, const float* d_B,
                                int32_t b_rows, int32_t b_ld, int32_t b_red_contig, int32_t red, int32_t a_ones_row,
                                float* d_work, float* d_C, int64_t sc_i, int64_t sc_j, int32_t splits, int64_t split_stride,
                                const float* d_bias, int32_t relu, void* stream) {
  const int ar = (int)(ceil_div(a_rows + 1, 128) * 128), br = (int)(ceil_div(b_rows, 256) * 256);
  const int rp = (int)(ceil_div(red, kPkKB) * kPkKB);
  float* a_hi = d_work; float* a_lo = a_hi + (int64_t)ar * rp;
  float* b_hi = a_lo + (int64_t)ar * rp; float* b_lo = b_hi + (int64_t)br * rp;
  PackBatch pb;
  memset(&pb, 0, sizeof(pb));
  int rc = pk_add_job(pb, d_A, a_ld, a_red_contig, a_rows, red, ar, rp, a_ones_row, a_hi, a_lo);
  if (rc != DZ_OK) return rc;
  rc = pk_add_job(pb, d_B, b_ld, b_red_contig, b_rows, red, br, rp, -1, b_hi, b_lo);
  if (rc != DZ_OK) return rc;
  rc = launch_pack("tc_pack_selftest", pb, stream);
  if (rc != DZ_OK) return rc;
  PkBatch kb;
  memset(&kb, 0, sizeof(kb));
  kb.n = 1;
  PkProblem& p = kb.p[0];
  p.A = PkOperand{a_hi, a_lo, ar / 8};
  p.B = PkOperand{b_hi, b_lo, br / 8};
  p.MI = a_rows + (a_ones_row >= 0 ? 1 : 0); p.NJ = b_rows; p.nkb = rp / kPkKB;
  p.C = d_C; p.sc_i = sc_i; p.sc_j = sc_j; p.splits = splits; p.split_stride = split_stride; p.bias_j = d_bias; p.relu = relu;
  return launch_pgemm("tc_pgemm_selftest", kb, stream);
}

// Self test of the IQN embedding epilogue (EPI 1): packs cos [M][latent] and embed_w [latent][D] as the learner's
// forward does, then runs the embedding problem of pk_embed_problem into the caller's images.
extern "C" int dz_test_iqn_embed_packed(const float* d_cos, int32_t M, int32_t latent, const float* d_embed_w, int32_t D,
                                        const float* d_bias, const float* d_mul, int32_t mul_div, int32_t mul_ld,
                                        float* d_work, float* d_e0, float* d_img_hi, float* d_img_lo, float* d_imgT_hi,
                                        float* d_imgT_lo, void* stream) {
  if (!d_cos || !d_embed_w || !d_bias || !d_mul || !d_work || !d_img_hi || !d_img_lo || (!d_imgT_hi != !d_imgT_lo))
    return fail(DZ_EINVAL, "test_iqn_embed_packed: NULL buffer");
  if (latent < 1 || latent > 8 * kPkKB) return fail(DZ_EINVAL, "test_iqn_embed_packed: latent must be in [1, 128]");
  if (M < 4 || M % 4 || D < 4 || D % 4) return fail(DZ_EINVAL, "test_iqn_embed_packed: M and D must be positive multiples of 4");
  if (mul_div < 1 || mul_ld < D || mul_ld % 4) return fail(DZ_EINVAL, "test_iqn_embed_packed: mul_div >= 1, mul_ld >= D and a multiple of 4");
  auto misaligned = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) != 0; };
  if (misaligned(d_bias) || misaligned(d_mul) || (d_e0 && misaligned(d_e0)))
    return fail(DZ_EINVAL, "test_iqn_embed_packed: bias, mul and e0 are read and written as float4");
  const int ar = (int)(ceil_div(M, 128) * 128), br = (int)(ceil_div(D, 256) * 256);
  const int rp = (int)(ceil_div(latent, kPkKB) * kPkKB);
  float* c_hi = d_work; float* c_lo = c_hi + (int64_t)ar * rp;
  float* w_hi = c_lo + (int64_t)ar * rp; float* w_lo = w_hi + (int64_t)br * rp;
  PackBatch pb;
  memset(&pb, 0, sizeof(pb));
  DZ_TRY(pk_add_job(pb, d_cos, latent, 1, M, latent, ar, rp, -1, c_hi, c_lo));
  DZ_TRY(pk_add_job(pb, d_embed_w, D, 0, D, latent, br, rp, -1, w_hi, w_lo));
  DZ_TRY(launch_pack("iqn_pack_selftest", pb, stream));
  PkBatch kb;
  memset(&kb, 0, sizeof(kb));
  kb.n = 1;
  const PkTarget img{d_img_hi, d_img_lo, ar / 8};
  const PkTarget imgT{d_imgT_hi, d_imgT_lo, (int)(ceil_div(D + 1, 128) * 128) / 8};
  kb.p[0] = pk_embed_problem(PkOperand{c_hi, c_lo, ar / 8}, PkOperand{w_hi, w_lo, br / 8}, M, D, rp / kPkKB, d_bias, d_mul,
                             mul_div, mul_ld, d_e0, img, imgT);
  return launch_pgemm("iqn_embed_selftest", kb, stream, 1);
}
