// Batched KV page copy: for every pool (one per layer) and every (src, dst) page pair, pool page src -> pool page dst, in
// one launch.  The copy-on-write of pages that several streams of a paged decode scope share (a forked prompt's partial
// page, a shared page a stream reaches again at a ring wrap).
//
// Work units are (pool, pair, part): each page is cut into `splits` equal parts of its access words, so that a copy of a
// few pairs still spreads over the grid, and the grid is bounded by the caller's `ctas`.  The access width is the
// largest of 16 / 8 / 4 / 1 bytes that divides the pool base and the page size (a page starts at base + index *
// page_bytes); every thread keeps UNROLL independent loads in flight before it stores.
#include "common.cuh"
#include "../../include/rstnet_b200.h"

#include <algorithm>
#include <new>
#include <vector>

namespace rstnet {
extern void count_launch();
}

namespace {

constexpr int kThreads = 256;
constexpr int kUnroll = 4;

struct Pools {
  char* p[RSTNET_KV_COPY_MAX_POOLS];
};

template <typename T>
__device__ __forceinline__ void copy_words(const char* src, char* dst, long long page_bytes, int part, int splits) {
  constexpr int W = (int)sizeof(T);
  const long long words = page_bytes / W;
  const long long lo = words * part / splits, hi = words * (part + 1) / splits;
  const T* s = reinterpret_cast<const T*>(src);
  T* d = reinterpret_cast<T*>(dst);
  for (long long v0 = lo + threadIdx.x; v0 < hi; v0 += (long long)kUnroll * blockDim.x) {
    T w[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const long long v = v0 + (long long)u * blockDim.x;
      if (v < hi) w[u] = s[v];
    }
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const long long v = v0 + (long long)u * blockDim.x;
      if (v < hi) d[v] = w[u];
    }
  }
}

__global__ void __launch_bounds__(kThreads) kv_pages_copy_kernel(const __grid_constant__ Pools pools, int n_pools,
                                                                 const int32_t* __restrict__ pairs, int n_pairs,
                                                                 long long page_bytes, int splits) {
  const long long units = (long long)n_pools * n_pairs * splits;
  for (long long u = blockIdx.x; u < units; u += gridDim.x) {
    const int part = (int)(u % splits);
    const long long pp = u / splits;
    const int pair = (int)(pp % n_pairs), pool = (int)(pp / n_pairs);
    const long long src = pairs[2 * pair], dst = pairs[2 * pair + 1];   // (the table may be pinned host memory)
    char* base = pools.p[pool];
    const unsigned long long a = (unsigned long long)(uintptr_t)base | (unsigned long long)page_bytes;
    const char* s = base + src * page_bytes;
    char* d = base + dst * page_bytes;
    if ((a & 15) == 0)
      copy_words<uint4>(s, d, page_bytes, part, splits);
    else if ((a & 7) == 0)
      copy_words<uint2>(s, d, page_bytes, part, splits);
    else if ((a & 3) == 0)
      copy_words<unsigned>(s, d, page_bytes, part, splits);
    else
      copy_words<unsigned char>(s, d, page_bytes, part, splits);
  }
}

// A page is the dst of at most one pair and never both a src and a dst, so the copies are independent of their order.
// Checked through sorted lists of the pages named: the work and memory depend on n_pairs only, not on the page indices.
int check_pairs(const int32_t* h, int n_pairs) {
  std::vector<int32_t> srcs((size_t)n_pairs), dsts((size_t)n_pairs);
  for (int i = 0; i < n_pairs; ++i) {
    RSTNET_REQUIRE(h[2 * i] >= 0 && h[2 * i + 1] >= 0, "kv_pages_copy: pair %d (%d -> %d) has a negative page", i, h[2 * i],
                   h[2 * i + 1]);
    RSTNET_REQUIRE(h[2 * i] != h[2 * i + 1], "kv_pages_copy: pair %d copies page %d onto itself", i, h[2 * i]);
    srcs[i] = h[2 * i];
    dsts[i] = h[2 * i + 1];
  }
  std::sort(srcs.begin(), srcs.end());
  std::sort(dsts.begin(), dsts.end());
  for (int i = 0; i < n_pairs; ++i) {
    RSTNET_REQUIRE(i == 0 || dsts[i] != dsts[i - 1], "kv_pages_copy: page %d is the dst of two pairs", dsts[i]);
    RSTNET_REQUIRE(!std::binary_search(srcs.begin(), srcs.end(), dsts[i]), "kv_pages_copy: page %d is both a src and a dst",
                   dsts[i]);
  }
  return 0;
}

}  // namespace

extern "C" int rstnet_kv_pages_copy(const void* const* pools, int32_t n_pools, const int32_t* pairs, int32_t n_pairs,
                                    int64_t page_bytes, int32_t ctas, rstnet_stream_t s) {
  RSTNET_REQUIRE(pools && pairs, "kv_pages_copy: null pools or pairs pointer");
  RSTNET_REQUIRE(n_pools >= 1 && n_pools <= RSTNET_KV_COPY_MAX_POOLS, "kv_pages_copy: n_pools = %d outside [1, %d]", n_pools,
                 RSTNET_KV_COPY_MAX_POOLS);
  RSTNET_REQUIRE(n_pairs >= 0, "kv_pages_copy: n_pairs = %d < 0", n_pairs);
  RSTNET_REQUIRE(page_bytes > 0, "kv_pages_copy: page_bytes = %lld <= 0", (long long)page_bytes);
  RSTNET_REQUIRE(ctas >= 1, "kv_pages_copy: ctas = %d < 1", ctas);
  Pools pp{};
  for (int i = 0; i < n_pools; ++i) {
    RSTNET_REQUIRE(pools[i], "kv_pages_copy: pool %d is a null pointer", i);
    pp.p[i] = static_cast<char*>(const_cast<void*>(pools[i]));
  }
  if (n_pairs == 0) return 0;
  // the pairs are checked on the host before the launch: a pinned host table directly, a device table through a
  // synchronous copy, which a stream that is capturing a graph cannot make
  cudaPointerAttributes at{};
  if (cudaPointerGetAttributes(&at, pairs) != cudaSuccess) cudaGetLastError();
  RSTNET_REQUIRE(at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeHost || at.type == cudaMemoryTypeManaged,
                 "kv_pages_copy: the pairs are neither device memory nor pinned host memory");
  // host vectors of n_pairs entries: an allocation failure is an error return, not an exception through the C ABI
  try {
    std::vector<int32_t> copy;
    const int32_t* h = pairs;
    if (at.type != cudaMemoryTypeHost) {
      cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
      RSTNET_REQUIRE(cudaStreamIsCapturing((cudaStream_t)s, &cap) == cudaSuccess && cap == cudaStreamCaptureStatusNone,
                     "kv_pages_copy: a device table cannot be checked while the stream captures a graph (pass pinned host pairs)");
      copy.resize(2 * (size_t)n_pairs);
      RSTNET_REQUIRE(cudaMemcpy(copy.data(), pairs, sizeof(int32_t) * 2 * (size_t)n_pairs, cudaMemcpyDeviceToHost) == cudaSuccess,
                     "kv_pages_copy: reading the pairs failed");
      h = copy.data();
    }
    if (int rc = check_pairs(h, n_pairs)) return rc;
  } catch (const std::bad_alloc&) {
    RSTNET_REQUIRE(false, "kv_pages_copy: out of host memory checking %d pairs", n_pairs);
  }
  const long long total = page_bytes * (long long)n_pools * n_pairs;
  const long long unit = std::max(1ll, total / (4ll * ctas));   // parts of about total / (4 * ctas) bytes
  long long splits = std::min(1024ll, std::max(1ll, (page_bytes + unit - 1) / unit));
  splits = std::max(1ll, std::min(splits, (1ll << 31) / ((long long)n_pools * n_pairs)));
  const long long units = (long long)n_pools * n_pairs * splits;
  const int grid = (int)std::min<long long>(ctas, units);
  kv_pages_copy_kernel<<<grid, kThreads, 0, (cudaStream_t)s>>>(pp, n_pools, pairs, n_pairs, (long long)page_bytes, (int)splits);
  rstnet::count_launch();
  return rstnet::check_launch("kv_pages_copy");
}
