#include "tmap.h"
#include <mutex>

namespace b200 {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, []() {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

static CUtensorMapSwizzle to_cu(Swz s) {
  switch (s) {
    case SWZ_32: return CU_TENSOR_MAP_SWIZZLE_32B;
    case SWZ_64: return CU_TENSOR_MAP_SWIZZLE_64B;
    case SWZ_128: return CU_TENSOR_MAP_SWIZZLE_128B;
    default: return CU_TENSOR_MAP_SWIZZLE_NONE;
  }
}

int make_act_map(CUtensorMap* out, const bf16* ptr, int N, int D, int H, int W, int C, int ld, int boxC, int boxW,
                 int boxH, int boxD, int estride, Swz swz, int vD, int vH, int vW) {
  EncodeTiledFn enc = get_encode();
  B200_REQUIRE(enc != nullptr, E_DRIVER, "cuTensorMapEncodeTiled not available (no CUDA driver?)");
  B200_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, E_INVALID, "activation pointer not 16B aligned");
  B200_REQUIRE((ld * 2) % 16 == 0, E_INVALID, "channel pitch %d not a multiple of 8 elements", ld);
  cuuint64_t dims[5] = {(cuuint64_t)C, (cuuint64_t)(vW > 0 ? vW : W), (cuuint64_t)(vH > 0 ? vH : H),
                        (cuuint64_t)(vD > 0 ? vD : D), (cuuint64_t)N};
  cuuint64_t strides[4] = {(cuuint64_t)ld * 2, (cuuint64_t)W * ld * 2, (cuuint64_t)H * W * ld * 2,
                           (cuuint64_t)D * H * W * ld * 2};
  cuuint32_t box[5] = {(cuuint32_t)boxC, (cuuint32_t)(boxW * estride), (cuuint32_t)(boxH * estride),
                       (cuuint32_t)(boxD * estride), 1};
  cuuint32_t es[5] = {1, (cuuint32_t)estride, (cuuint32_t)estride, (cuuint32_t)estride, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<bf16*>(ptr), dims, strides, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, to_cu(swz), CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  B200_REQUIRE(r == CUDA_SUCCESS, E_DRIVER,
               "cuTensorMapEncodeTiled(act) failed: %d (N%d D%d H%d W%d C%d ld%d box %d,%d,%d,%d es%d swz%d)", (int)r,
               N, D, H, W, C, ld, boxC, boxW, boxH, boxD, estride, (int)swz);
  return OK;
}

int make_act_map_class(CUtensorMap* out, const bf16* ptr, int N, int D, int H, int W, int C, int ld, int pd, int ph, int pw,
                       int boxC, int boxW, int boxH, int boxD, Swz swz) {
  EncodeTiledFn enc = get_encode();
  B200_REQUIRE(enc != nullptr, E_DRIVER, "cuTensorMapEncodeTiled not available (no CUDA driver?)");
  B200_REQUIRE(D % 2 == 0 && H % 2 == 0 && W % 2 == 0, E_INVALID, "class map: extents %dx%dx%d must be even", D, H, W);
  const bf16* base = ptr + (((long long)pd * H + ph) * W + pw) * ld;
  B200_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0 && (ld * 2) % 16 == 0, E_INVALID, "class map: misaligned view");
  cuuint64_t dims[5] = {(cuuint64_t)C, (cuuint64_t)(W / 2), (cuuint64_t)(H / 2), (cuuint64_t)(D / 2), (cuuint64_t)N};
  cuuint64_t strides[4] = {(cuuint64_t)2 * ld * 2, (cuuint64_t)2 * W * ld * 2, (cuuint64_t)2 * H * W * ld * 2,
                           (cuuint64_t)D * H * W * ld * 2};
  cuuint32_t box[5] = {(cuuint32_t)boxC, (cuuint32_t)boxW, (cuuint32_t)boxH, (cuuint32_t)boxD, 1};
  cuuint32_t es[5] = {1, 1, 1, 1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<bf16*>(base), dims, strides, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, to_cu(swz), CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  B200_REQUIRE(r == CUDA_SUCCESS, E_DRIVER, "cuTensorMapEncodeTiled(class) failed: %d (N%d D%d H%d W%d C%d ld%d p%d%d%d)", (int)r, N,
               D, H, W, C, ld, pd, ph, pw);
  return OK;
}

int make_act_map_classpair(CUtensorMap* out, const bf16* ptr, int N, int D, int H, int W, int C, int ld, int pd, int ph, int boxC,
                           int boxW, int boxH, int boxD, Swz swz) {
  EncodeTiledFn enc = get_encode();
  B200_REQUIRE(enc != nullptr, E_DRIVER, "cuTensorMapEncodeTiled not available (no CUDA driver?)");
  B200_REQUIRE(D % 2 == 0 && H % 2 == 0 && W % 2 == 0, E_INVALID, "class-pair map: extents %dx%dx%d must be even", D, H, W);
  const bf16* base = ptr + (((long long)pd * H + ph) * W) * ld;
  B200_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0 && (ld * 2) % 16 == 0, E_INVALID, "class-pair map: misaligned view");
  cuuint64_t dims[5] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)(H / 2), (cuuint64_t)(D / 2), (cuuint64_t)N};
  cuuint64_t strides[4] = {(cuuint64_t)ld * 2, (cuuint64_t)2 * W * ld * 2, (cuuint64_t)2 * H * W * ld * 2, (cuuint64_t)D * H * W * ld * 2};
  cuuint32_t box[5] = {(cuuint32_t)boxC, (cuuint32_t)boxW, (cuuint32_t)boxH, (cuuint32_t)boxD, 1};
  cuuint32_t es[5] = {1, 1, 1, 1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<bf16*>(base), dims, strides, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, to_cu(swz), CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  B200_REQUIRE(r == CUDA_SUCCESS, E_DRIVER, "cuTensorMapEncodeTiled(class pair) failed: %d (N%d D%d H%d W%d C%d ld%d p%d%d)", (int)r, N, D,
               H, W, C, ld, pd, ph);
  return OK;
}

int make_w_map(CUtensorMap* out, const bf16* ptr, int T, int R, int K, int boxK, int boxR, Swz swz, int boxT) {
  EncodeTiledFn enc = get_encode();
  B200_REQUIRE(enc != nullptr, E_DRIVER, "cuTensorMapEncodeTiled not available (no CUDA driver?)");
  B200_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, E_INVALID, "weight pointer not 16B aligned");
  B200_REQUIRE((K * 2) % 16 == 0, E_INVALID, "packed weight K=%d not a multiple of 8", K);
  cuuint64_t dims[3] = {(cuuint64_t)K, (cuuint64_t)R, (cuuint64_t)T};
  cuuint64_t strides[2] = {(cuuint64_t)K * 2, (cuuint64_t)R * K * 2};
  cuuint32_t box[3] = {(cuuint32_t)boxK, (cuuint32_t)boxR, (cuuint32_t)boxT};
  cuuint32_t es[3] = {1, 1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<bf16*>(ptr), dims, strides, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, to_cu(swz), CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  B200_REQUIRE(r == CUDA_SUCCESS, E_DRIVER, "cuTensorMapEncodeTiled(w) failed: %d (T%d R%d K%d box %d,%d swz%d)",
               (int)r, T, R, K, boxK, boxR, (int)swz);
  return OK;
}

}  // namespace b200
