// Library-wide runtime bits: launch counter, version, tensor-map encoding through the driver
// entry point (resolved lazily so the .so loads on a machine without libcuda / without a GPU).
#include "alm_common.cuh"

namespace alm {

unsigned long long g_launch_count = 0;

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn resolve_encode() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

int make_tensor_map(CUtensorMap* out, const void* base, int elem_bytes, int rank, const uint64_t* dims,
                    const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes) {
  EncodeTiledFn enc = resolve_encode();
  if (!enc) {
    fprintf(stderr, "[alm] cuTensorMapEncodeTiled unavailable (no CUDA driver?)\n");
    return ALM_ERR_CUDA;
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15u) != 0) {
    fprintf(stderr, "[alm] tensor map base %p is not 16-B aligned\n", base);
    return ALM_ERR_ALIGN;
  }
  cuuint64_t gdim[5];
  cuuint64_t gstr[5];
  cuuint32_t bdim[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
    estr[i] = 1;
    if (i > 0) {
      gstr[i - 1] = strides_bytes[i];
      if (strides_bytes[i] % 16 != 0) {
        fprintf(stderr, "[alm] tensor map stride %llu (dim %d) is not a multiple of 16 B\n",
                (unsigned long long)strides_bytes[i], i);
        return ALM_ERR_ALIGN;
      }
    }
  }
  if (swizzle_bytes != 0 && swizzle_bytes != 64 && swizzle_bytes != 128) return ALM_ERR_ARG;
  const CUtensorMapSwizzle swz = swizzle_bytes == 128  ? CU_TENSOR_MAP_SWIZZLE_128B
                                 : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                                       : CU_TENSOR_MAP_SWIZZLE_NONE;
  CUtensorMapDataType dt = elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  CUresult r = enc(out, dt, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bdim, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fprintf(stderr, "[alm] cuTensorMapEncodeTiled failed with %d (rank %d dims %llu,%llu,%llu box %u,%u,%u)\n", (int)r,
            rank, (unsigned long long)gdim[0], (unsigned long long)(rank > 1 ? gdim[1] : 0),
            (unsigned long long)(rank > 2 ? gdim[2] : 0), bdim[0], rank > 1 ? bdim[1] : 0, rank > 2 ? bdim[2] : 0);
    return ALM_ERR_CUDA;
  }
  return ALM_OK;
}

}  // namespace alm

extern "C" {

int alm_version(void) { return 100; }

unsigned long long alm_launch_count(void) { return alm::g_launch_count; }

void alm_reset_launch_count(void) { alm::g_launch_count = 0; }

const char* alm_status_string(int code) {
  switch (code) {
    case ALM_OK: return "ok";
    case ALM_ERR_ARG: return "invalid argument";
    case ALM_ERR_ALIGN: return "pointer or stride not aligned as the kernel requires";
    case ALM_ERR_CUDA: return "CUDA runtime/driver error (see stderr)";
    case ALM_ERR_UNSUPPORTED: return "shape or mode not supported by this build";
    default: return "unknown status";
  }
}

}  // extern "C"
