// Device-resident columnar batch model (HBM layout) of the engine.
//
// Layout = Arrow's, as delivered at the ExecutionPlan boundary (SURVEY.md 8 "Conventions"):
//   fixed width  : values buffer, `width` bytes per row (Decimal128: 16-byte LE two's complement)
//   Utf8         : int32 offsets (n+1) + chars                                  [PH_UTF8]
//   Utf8 (intermediate results): 16-byte views {ptr,len} into kept-alive chars  [PH_STRVIEW]
//   Bool         : one byte per value on device (Arrow bitmaps are expanded at ingest / packed at export)
//   validity     : one byte per row, nullptr == no NULLs
// Every allocation carries >= 64 bytes of slack so that 16-byte-granular TMA bulk copies of the
// last tile never leave the allocation.
#pragma once
#include <cuda_runtime.h>

#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../../include/b200exec.h"
#include "../common/plan.hpp"
#include "../device/program.h"

namespace b200 {

struct EngineError : std::runtime_error {
  int code;
  EngineError(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

#define CUDA_CHECK(expr)                                                                                      \
  do {                                                                                                        \
    cudaError_t _e = (expr);                                                                                  \
    if (_e != cudaSuccess)                                                                                    \
      throw EngineError(_e == cudaErrorMemoryAllocation ? B200_ERR_OOM : B200_ERR_CUDA,                       \
                        std::string("CUDA error: ") + cudaGetErrorString(_e) + " at " + __FILE__ + ":" +      \
                            std::to_string(__LINE__));                                                        \
  } while (0)

// Small allocations (status words, offsets of a few rows, literal pools, the 4-row batches at the tail of a query) are
// carved out of per-thread 2 MB chunks instead of each paying a cudaMallocAsync / cudaFreeAsync pair: a stage issues
// dozens of them, and at the tail of a query the driver calls cost more than the kernels.  A chunk is stream-ordered
// like the allocations it replaces (allocated and freed on the stream that uses it) and lives until the last
// sub-allocation is released.
struct ArenaChunk {
  uint8_t* base = nullptr;
  size_t cap = 0, used = 0;
  cudaStream_t stream = nullptr;
  ~ArenaChunk() {
    if (base) cudaFreeAsync(base, stream);
  }
};
static const size_t ARENA_CHUNK_BYTES = (size_t)2 << 20;
static const size_t ARENA_MAX_ALLOC = (size_t)64 << 10;
// the chunk the calling thread carves new small allocations from
inline std::shared_ptr<ArenaChunk>& arena_chunk() {
  static thread_local std::shared_ptr<ArenaChunk> cur;
  return cur;
}

struct DevAlloc {
  void* ptr = nullptr;
  size_t bytes = 0;
  cudaStream_t stream = nullptr;
  std::shared_ptr<ArenaChunk> chunk;  // set for arena sub-allocations
  DevAlloc(size_t n, cudaStream_t st) : bytes(n), stream(st) {
    const size_t padded = ((n + 255) & ~(size_t)255) + 256;
    if (padded <= ARENA_MAX_ALLOC) {
      std::shared_ptr<ArenaChunk>& cur = arena_chunk();
      if (!cur || cur->stream != st || cur->used + padded > cur->cap) {
        auto c = std::make_shared<ArenaChunk>();
        void* p = nullptr;
        CUDA_CHECK(cudaMallocAsync(&p, ARENA_CHUNK_BYTES, st));
        c->base = (uint8_t*)p;
        c->cap = ARENA_CHUNK_BYTES;
        c->stream = st;
        cur = c;
      }
      ptr = cur->base + cur->used;
      cur->used += padded;
      chunk = cur;
      return;
    }
    CUDA_CHECK(cudaMallocAsync(&ptr, padded, st));
  }
  ~DevAlloc() {
    if (ptr && !chunk) cudaFreeAsync(ptr, stream);
  }
  DevAlloc(const DevAlloc&) = delete;
  DevAlloc& operator=(const DevAlloc&) = delete;
};
typedef std::shared_ptr<DevAlloc> DevPtr;

inline DevPtr dev_alloc(size_t n, cudaStream_t st) { return std::make_shared<DevAlloc>(n, st); }

inline Phys phys_of(const DataType& t) {
  switch (t.id) {
    case TypeId::Bool: return PH_BOOL8;
    case TypeId::Int8: return PH_I8;
    case TypeId::Int16: return PH_I16;
    case TypeId::Int32:
    case TypeId::Date32: return PH_I32;
    case TypeId::Int64:
    case TypeId::Timestamp: return PH_I64;
    case TypeId::UInt8: return PH_U8;
    case TypeId::UInt16: return PH_U16;
    case TypeId::UInt32: return PH_U32;
    case TypeId::UInt64: return PH_U64;
    case TypeId::Float32: return PH_F32;
    case TypeId::Float64: return PH_F64;
    case TypeId::Decimal128: return PH_DEC128;
    case TypeId::Utf8: return PH_UTF8;
    default: return PH_U8;
  }
}
inline int phys_width(Phys p) {
  switch (p) {
    case PH_I8:
    case PH_U8:
    case PH_BOOL8: return 1;
    case PH_I16:
    case PH_U16: return 2;
    case PH_I32:
    case PH_U32:
    case PH_F32:
    case PH_UTF8: return 4;
    case PH_DEC128:
    case PH_STRVIEW: return 16;
    default: return 8;
  }
}
inline VK vk_of(const DataType& t) { return (VK)(int)t.pk(); }

struct DevColumn {
  std::string name;
  DataType type;
  bool nullable = true;
  Phys phys = PH_I64;
  int64_t n = 0;
  const uint8_t* data = nullptr;   // values / offsets / views (may point inside an allocation: slices)
  const uint8_t* valid = nullptr;  // byte per row or nullptr
  const uint8_t* chars = nullptr;  // PH_UTF8 only
  int64_t chars_bytes = -1;        // PH_UTF8: bytes referenced by this column's rows (-1 unknown)
  // 4-byte image of every row, or nullptr (build_column_images; kept alive through `keep`): PH_UTF8 with only <= 3-byte
  // strings: len << 24 | bytes; PH_DEC128 whose values all fit int32: the value as int32
  const uint32_t* img32 = nullptr;
  std::vector<DevPtr> keep;        // allocations that must outlive this column
  int width() const { return phys_width(phys); }
};

struct DevBatch {
  std::vector<DevColumn> cols;
  int64_t n = 0;
};
typedef std::shared_ptr<DevBatch> DevBatchPtr;

// row slice [r0, r1) of a column (zero copy)
inline DevColumn slice_column(const DevColumn& c, int64_t r0, int64_t r1) {
  DevColumn o = c;
  o.n = r1 - r0;
  o.data = c.data ? c.data + r0 * c.width() : nullptr;
  o.valid = c.valid ? c.valid + r0 : nullptr;
  o.img32 = c.img32 ? c.img32 + r0 : nullptr;
  o.chars_bytes = -1;
  return o;
}

}  // namespace b200
