// Segment gather / scatter: move one batch row's streaming state between its device buffers and a packed staging blob
// (pinned host memory reached through UVA), in one launch per direction (session suspend / resume, serve.py).
//
// A segment is `count` pieces of `bytes` at base + i * stride_bytes; it occupies staging[staging_offset, + count * bytes)
// with the pieces back to back.  Each CTA walks work units (segment, part): a segment is cut into `splits` equal parts of
// its access words so that a few large segments still spread over the grid, and the grid is bounded by the caller's
// `ctas` so that a swap on a side stream leaves the remaining SMs to the decode step beside it.  The access width is the
// largest of 16 / 8 / 4 / 1 bytes that divides the base, stride, piece size and staging address of the segment; every
// thread keeps UNROLL independent loads in flight before it stores, so that reads over the host link are not latency-bound.
#include "common.cuh"
#include "../../include/rstnet_b200.h"

#include <algorithm>
#include <utility>
#include <vector>

namespace rstnet {
extern void count_launch();
}

namespace {

constexpr int kThreads = 256;
constexpr int kUnroll = 4;

template <typename T>
__device__ __forceinline__ void move_words(const rstnet_segment& sg, char* staging, int part, int splits, bool gather) {
  constexpr int W = (int)sizeof(T);
  const long long vpp = sg.bytes / W;                       // words per piece
  const long long total = vpp * (long long)sg.count;
  const long long lo = total * part / splits, hi = total * (part + 1) / splits;
  char* dev = static_cast<char*>(sg.base);
  T* stg = reinterpret_cast<T*>(staging + sg.staging_offset);
  for (long long v0 = lo + threadIdx.x; v0 < hi; v0 += (long long)kUnroll * blockDim.x) {
    T w[kUnroll];
    T* dst[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const long long v = v0 + (long long)u * blockDim.x;
      dst[u] = nullptr;
      if (v < hi) {
        const long long piece = vpp == total ? 0 : v / vpp;
        T* d = reinterpret_cast<T*>(dev + piece * sg.stride_bytes) + (v - piece * vpp);
        if (gather) {
          w[u] = *d;
          dst[u] = stg + v;
        } else {
          w[u] = stg[v];
          dst[u] = d;
        }
      }
    }
#pragma unroll
    for (int u = 0; u < kUnroll; ++u)
      if (dst[u]) *dst[u] = w[u];
  }
}

__global__ void __launch_bounds__(kThreads) segments_kernel(const rstnet_segment* __restrict__ table, int n, int splits,
                                                            char* staging, int gather) {
  __shared__ rstnet_segment sg;
  const long long units = (long long)n * splits;
  for (long long u = blockIdx.x; u < units; u += gridDim.x) {
    __syncthreads();                                        // the previous unit's readers are done with `sg`
    if (threadIdx.x == 0) sg = table[u / splits];           // one read of the entry (the table may be host memory)
    __syncthreads();
    const int part = (int)(u % splits);
    if (sg.count == 0 || sg.bytes == 0) continue;
    const unsigned long long a = (unsigned long long)(uintptr_t)sg.base | (unsigned long long)sg.stride_bytes |
                                 (unsigned long long)sg.bytes | (unsigned long long)(uintptr_t)(staging + sg.staging_offset);
    if ((a & 15) == 0)
      move_words<uint4>(sg, staging, part, splits, gather);
    else if ((a & 7) == 0)
      move_words<uint2>(sg, staging, part, splits, gather);
    else if ((a & 3) == 0)
      move_words<unsigned>(sg, staging, part, splits, gather);
    else
      move_words<unsigned char>(sg, staging, part, splits, gather);
  }
}

// memory the device can address: device memory or registered (pinned / mapped) host memory
bool device_addressable(const void* p, bool* on_host) {
  cudaPointerAttributes at{};
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  *on_host = at.type == cudaMemoryTypeHost;
  return at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeHost || at.type == cudaMemoryTypeManaged;
}

int segments_run(const rstnet_segment* table, int32_t n, void* staging, int32_t ctas, rstnet_stream_t s, bool gather) {
  const char* what = gather ? "segments_gather" : "segments_scatter";
  RSTNET_REQUIRE(n >= 0, "%s: n = %d < 0", what, n);
  RSTNET_REQUIRE(ctas >= 1, "%s: ctas = %d < 1", what, ctas);
  if (n == 0) return 0;
  RSTNET_REQUIRE(table && staging, "%s: null table or staging pointer", what);
  bool table_host = false, staging_host = false;
  RSTNET_REQUIRE(device_addressable(table, &table_host), "%s: the table is neither device memory nor pinned host memory", what);
  RSTNET_REQUIRE(device_addressable(staging, &staging_host), "%s: staging is neither pinned host memory nor device memory", what);
  // every entry is checked on the host before the launch: a host table directly, a device table through a copy
  std::vector<rstnet_segment> copy;
  const rstnet_segment* h = table;
  if (!table_host) {
    copy.resize((size_t)n);
    RSTNET_REQUIRE(cudaMemcpy(copy.data(), table, sizeof(rstnet_segment) * (size_t)n, cudaMemcpyDeviceToHost) == cudaSuccess,
                   "%s: reading the segment table failed", what);
    h = copy.data();
  }
  std::vector<std::pair<long long, long long>> ranges;
  ranges.reserve((size_t)n);
  long long max_len = 0, total = 0;
  for (int i = 0; i < n; ++i) {
    const rstnet_segment& g = h[i];
    RSTNET_REQUIRE(g.base, "%s: segment %d has a null base", what, i);
    RSTNET_REQUIRE(g.count >= 0 && g.bytes >= 0 && g.staging_offset >= 0, "%s: segment %d has count %d, bytes %lld, staging "
                   "offset %lld (each must be >= 0)", what, i, g.count, (long long)g.bytes, (long long)g.staging_offset);
    RSTNET_REQUIRE(g.count == 0 || g.bytes <= (1ll << 62) / g.count, "%s: segment %d is too large", what, i);
    const long long len = g.bytes * (long long)g.count;
    if (!gather && g.count > 1)
      RSTNET_REQUIRE(g.stride_bytes >= g.bytes || g.stride_bytes <= -g.bytes, "%s: the pieces of segment %d overlap (stride "
                     "%lld, %lld bytes each)", what, i, (long long)g.stride_bytes, (long long)g.bytes);
    if (len == 0) continue;
    RSTNET_REQUIRE(g.staging_offset <= (1ll << 62) - len, "%s: segment %d lies past the staging address range", what, i);
    ranges.emplace_back(g.staging_offset, g.staging_offset + len);
    max_len = std::max(max_len, len);
    total += len;
  }
  std::sort(ranges.begin(), ranges.end());
  for (size_t i = 1; i < ranges.size(); ++i)
    RSTNET_REQUIRE(ranges[i].first >= ranges[i - 1].second, "%s: two segments overlap in staging ([%lld, %lld) and [%lld, %lld))",
                   what, ranges[i - 1].first, ranges[i - 1].second, ranges[i].first, ranges[i].second);
  if (total == 0) return 0;
  // parts per segment: the largest segment is cut into parts of about total / (4 * ctas) bytes
  const long long unit = std::max(1ll, total / (4ll * ctas));
  long long splits = std::min(1024ll, std::max(1ll, (max_len + unit - 1) / unit));
  splits = std::max(1ll, std::min(splits, (1ll << 31) / n));
  const long long units = (long long)n * splits;
  const int grid = (int)std::min<long long>(ctas, units);
  segments_kernel<<<grid, kThreads, 0, (cudaStream_t)s>>>(table, n, (int)splits, static_cast<char*>(staging), gather ? 1 : 0);
  rstnet::count_launch();
  return rstnet::check_launch(what);
}

}  // namespace

extern "C" int rstnet_segments_gather(const rstnet_segment* table_dev, int32_t n, void* staging, int32_t ctas, rstnet_stream_t s) {
  return segments_run(table_dev, n, staging, ctas, s, true);
}

extern "C" int rstnet_segments_scatter(const rstnet_segment* table_dev, int32_t n, const void* staging, int32_t ctas,
                                       rstnet_stream_t s) {
  return segments_run(table_dev, n, const_cast<void*>(staging), ctas, s, false);
}
