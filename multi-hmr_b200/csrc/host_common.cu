// Host-side utilities shared by all translation units of libmhmr_sm90.so.
#include <cstdlib>
#include "common.cuh"

#include <algorithm>
#include <mutex>

namespace mhmr {

namespace {
thread_local std::string g_last_error;
}

void set_last_error(const std::string& msg) { g_last_error = msg; }
const char* get_last_error() { return g_last_error.c_str(); }

namespace {
using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                   const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                   const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    // Resolved at run time through the runtime: no link-time dependency on libcuda.so, so the
    // library loads (and its exports can be checked) on hosts without a driver.
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) ==
            cudaSuccess &&
        qres == cudaDriverEntryPointSuccess) {
      fn = reinterpret_cast<EncodeTiledFn>(p);
    }
  });
  return fn;
}
}  // namespace

int make_tmap_2d(CUtensorMap* out, const void* gptr, CUtensorMapDataType dtype, int elem_bytes,
                 uint64_t rows, uint64_t cols, uint64_t pitch_bytes, uint32_t box_rows,
                 uint32_t box_cols, bool swizzle128) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) {
    set_last_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    return MHMR_ERR_CUDA;
  }
  if (swizzle128 && box_cols * static_cast<uint32_t>(elem_bytes) != 128u) {
    set_last_error("make_tmap_2d: 128B swizzle needs a 128-byte inner box");
    return MHMR_ERR_ARG;
  }
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {pitch_bytes};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, dtype, 2, const_cast<void*>(gptr), gdim, gstride, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed with CUresult " + std::to_string(static_cast<int>(r)) +
                   " (rows=" + std::to_string(rows) + " cols=" + std::to_string(cols) +
                   " pitch=" + std::to_string(pitch_bytes) + ")");
    return MHMR_ERR_CUDA;
  }
  return MHMR_OK;
}

int make_tmap_3d(CUtensorMap* out, const void* gptr, CUtensorMapDataType dtype, int elem_bytes,
                 uint64_t depth, uint64_t rows, uint64_t cols, uint64_t depth_pitch_bytes, uint64_t pitch_bytes,
                 uint32_t box_rows, uint32_t box_cols, bool swizzle128) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) {
    set_last_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    return MHMR_ERR_CUDA;
  }
  if (swizzle128 && box_cols * static_cast<uint32_t>(elem_bytes) != 128u) {
    set_last_error("make_tmap_3d: 128B swizzle needs a 128-byte inner box");
    return MHMR_ERR_ARG;
  }
  cuuint64_t gdim[3] = {cols, rows, depth};
  cuuint64_t gstride[2] = {pitch_bytes, depth_pitch_bytes};
  cuuint32_t box[3] = {box_cols, box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(out, dtype, 3, const_cast<void*>(gptr), gdim, gstride, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled (3-D) failed with CUresult " + std::to_string(static_cast<int>(r)) +
                   " (depth=" + std::to_string(depth) + " rows=" + std::to_string(rows) +
                   " cols=" + std::to_string(cols) + " pitch=" + std::to_string(pitch_bytes) + ")");
    return MHMR_ERR_CUDA;
  }
  return MHMR_OK;
}

bool PerDeviceOnce::first() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return true;
  if (done[dev]) return false;
  done[dev] = true;
  return true;
}

int device_sm_count() {
  static int sms[64] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (sms[dev] == 0) {
    if (cudaDeviceGetAttribute(&sms[dev], cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms[dev] <= 0)
      sms[dev] = 132;
  }
  return sms[dev];
}

CallScratch::~CallScratch() {
  if (base_ != nullptr) cudaFreeAsync(base_, st_);
}

size_t CallScratch::region(size_t bytes, bool staged) {
  size_t& end = staged ? staged_bytes_ : device_bytes_;
  regions_.push_back({end, staged});
  end += align256(bytes);
  if (staged) blob_.resize(staged_bytes_);
  return regions_.size() - 1;
}

int CallScratch::allocate() {
  const size_t bytes = std::max<size_t>(staged_bytes_ + device_bytes_, 256);
  MHMR_CUDA_CHECK(cudaMallocAsync(reinterpret_cast<void**>(&base_), bytes, st_));
  return MHMR_OK;
}

int CallScratch::upload() {
  if (staged_bytes_ > 0) MHMR_CUDA_CHECK(cudaMemcpyAsync(base_, blob_.data(), staged_bytes_, cudaMemcpyHostToDevice, st_));
  return MHMR_OK;
}

int CallScratch::release() {
  uint8_t* p = base_;
  base_ = nullptr;
  if (p != nullptr) MHMR_CUDA_CHECK(cudaFreeAsync(p, st_));
  return MHMR_OK;
}

bool pdl_enabled() {
  static int on = -1;
  if (on < 0) {
    const char* e = std::getenv("MHMR_PDL");
    on = (e != nullptr && e[0] == '0') ? 0 : 1;
  }
  return on == 1;
}

}  // namespace mhmr
