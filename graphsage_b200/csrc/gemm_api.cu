// gs_sage_gemm: argument checking and dispatch over gs_math.
#include "common.cuh"

namespace gs {
int32_t sage_gemm_simt(int64_t M, const gs_gemm_part* parts, const gs_gemm_row_ids* row_ids, int32_t n_parts,
                       int32_t combine, const float* bias, int32_t act, float* out, int64_t ldo, cudaStream_t st);
int64_t sage_gemm_tc_workspace(int64_t M, const gs_gemm_part* parts, int32_t n_parts, int32_t math);
int32_t sage_gemm_tc(int64_t M, const gs_gemm_part* parts, const gs_gemm_row_ids* row_ids, int32_t n_parts, int32_t combine,
                     const float* bias, int32_t act, int32_t math, float* out, int64_t ldo, const void* workspace,
                     cudaStream_t st);
int32_t sage_gemm_tc_pack(const gs_gemm_part* parts, int32_t n_parts, int32_t math, void* workspace, cudaStream_t st);
}  // namespace gs

static int32_t check_parts(int64_t M, const gs_gemm_part* parts, int32_t n_parts, int32_t combine, bool need_a = true) {
  GS_REQUIRE(M >= 0, "gs_sage_gemm: M < 0");
  GS_REQUIRE(parts && (n_parts == 1 || n_parts == 2), "gs_sage_gemm: n_parts must be 1 or 2 (got %d)", n_parts);
  GS_REQUIRE(combine == GS_COMBINE_ADD || combine == GS_COMBINE_CONCAT, "gs_sage_gemm: combine=%d", combine);
  for (int i = 0; i < n_parts; ++i) {
    GS_REQUIRE(parts[i].K >= 1 && parts[i].N >= 1, "gs_sage_gemm: part %d has K=%d N=%d", i, parts[i].K, parts[i].N);
    GS_REQUIRE(parts[i].lda >= parts[i].K && parts[i].ldb >= parts[i].N, "gs_sage_gemm: part %d leading dims too small", i);
    GS_REQUIRE(M == 0 || ((parts[i].A || !need_a) && parts[i].B), "gs_sage_gemm: part %d NULL operand", i);
  }
  if (n_parts == 2 && combine == GS_COMBINE_ADD)
    GS_REQUIRE(parts[0].N == parts[1].N, "gs_sage_gemm: ADD needs equal N (%d vs %d)", parts[0].N, parts[1].N);
  return GS_OK;
}

extern "C" {

int64_t gs_sage_gemm_workspace_bytes(int64_t M, const gs_gemm_part* parts_host, int32_t n_parts, int32_t math) {
  if (!parts_host || n_parts < 1 || n_parts > 2 || M < 0) return -1;
  if (math == GS_MATH_FP32_SIMT) return 0;
  return gs::sage_gemm_tc_workspace(M, parts_host, n_parts, math);
}

static bool is_tc(int32_t math) { return math == GS_MATH_TF32X3 || math == GS_MATH_TF32 || math == GS_MATH_BF16; }

int32_t gs_sage_gemm_pack(const gs_gemm_part* parts_host, int32_t n_parts, int32_t math, void* workspace, void* stream) {
  int32_t rc = check_parts(1, parts_host, n_parts, GS_COMBINE_CONCAT, false);   // packing reads the B matrices only
  if (rc != GS_OK) return rc;
  if (math == GS_MATH_FP32_SIMT) return GS_OK;      // nothing to pack
  GS_REQUIRE(is_tc(math), "gs_sage_gemm_pack: unknown math mode %d", math);
  return gs::sage_gemm_tc_pack(parts_host, n_parts, math, workspace, (cudaStream_t)stream);
}

int32_t gs_sage_gemm_rows(int64_t M, const gs_gemm_part* parts_host, const gs_gemm_row_ids* row_ids_host, int32_t n_parts,
                          int32_t combine, const float* bias, int32_t act, int32_t math, float* out, int64_t ldo,
                          const void* workspace, void* stream) {
  int32_t rc = check_parts(M, parts_host, n_parts, combine);
  if (rc != GS_OK) return rc;
  gs_gemm_row_ids rid[2];
  memset(rid, 0, sizeof(rid));
  for (int i = 0; row_ids_host && i < n_parts; ++i) {
    const gs_gemm_row_ids& R = row_ids_host[i];
    if (R.n_ranges == 0) continue;
    GS_REQUIRE(R.n_ranges > 0 && R.n_ranges <= GS_MAX_SEGMENTS, "gs_sage_gemm_rows: part %d has n_ranges=%d (max %d)", i,
               R.n_ranges, GS_MAX_SEGMENTS);
    GS_REQUIRE(R.n_table_rows >= 1 && R.n_table_rows < ((int64_t)1 << 31), "gs_sage_gemm_rows: part %d n_table_rows=%lld", i,
               (long long)R.n_table_rows);
    for (int s = 0; s < R.n_ranges; ++s)
      GS_REQUIRE(R.ranges[s].n >= 0 && R.ranges[s].row0 >= 0 && (R.ranges[s].ids || R.ranges[s].n == 0),
                 "gs_sage_gemm_rows: part %d range %d is invalid", i, s);
    rid[i] = R;
  }
  if (M == 0) return GS_OK;
  GS_REQUIRE(out, "gs_sage_gemm: out is NULL");
  int ntot = parts_host[0].N + ((n_parts == 2 && combine == GS_COMBINE_CONCAT) ? parts_host[1].N : 0);
  GS_REQUIRE(ldo >= ntot, "gs_sage_gemm: ldo=%lld < output width %d", (long long)ldo, ntot);
  GS_REQUIRE(act == GS_ACT_NONE || act == GS_ACT_RELU, "gs_sage_gemm: act=%d", act);
  if (math == GS_MATH_FP32_SIMT)
    return gs::sage_gemm_simt(M, parts_host, rid, n_parts, combine, bias, act, out, ldo, (cudaStream_t)stream);
  GS_REQUIRE(is_tc(math), "gs_sage_gemm: unknown math mode %d", math);
  return gs::sage_gemm_tc(M, parts_host, rid, n_parts, combine, bias, act, math, out, ldo, workspace, (cudaStream_t)stream);
}

int32_t gs_sage_gemm_prepacked(int64_t M, const gs_gemm_part* parts_host, int32_t n_parts, int32_t combine,
                               const float* bias, int32_t act, int32_t math, float* out, int64_t ldo,
                               const void* workspace, void* stream) {
  return gs_sage_gemm_rows(M, parts_host, nullptr, n_parts, combine, bias, act, math, out, ldo, workspace, stream);
}

int32_t gs_sage_gemm(int64_t M, const gs_gemm_part* parts_host, int32_t n_parts, int32_t combine, const float* bias,
                     int32_t act, int32_t math, float* out, int64_t ldo, void* workspace, void* stream) {
  if (M > 0 && math != GS_MATH_FP32_SIMT) {
    int32_t rc = gs_sage_gemm_pack(parts_host, n_parts, math, workspace, stream);
    if (rc != GS_OK) return rc;
  }
  return gs_sage_gemm_prepacked(M, parts_host, n_parts, combine, bias, act, math, out, ldo, workspace, stream);
}

}  // extern "C"
