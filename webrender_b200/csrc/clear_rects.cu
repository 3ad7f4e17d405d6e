// clear_rects.cu — the rect-list clear kernels (see clear_rects.cuh), a translation unit of their own.
#include "clear_rects.cuh"

// the last rect whose first row is <= g
__device__ __forceinline__ int wr_clear_rect_of_row(const ClearRects& p, int g) {
  int lo = 0, hi = p.n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (p.row0[mid] <= g) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// A row as wr_clear_u32 writes it: 16-byte vectors on 4-pixel boundaries, the head and tail by column slice 0.
__global__ void wr_clear_rects_u32(const __grid_constant__ ClearRects p) {
  const int g = blockIdx.x, i = wr_clear_rect_of_row(p, g);
  const int4 r = p.r[i];
  const int x0 = r.x, x1 = r.z, y = r.y + (g - p.row0[i]);
  const uint32_t v = p.v;
  uint32_t* row = (uint32_t*)(p.base + (size_t)y * p.pitch);
  int xa = (x0 + 3) & ~3, xb = x1 & ~3;
  if (xa >= xb) {
    for (int x = x0 + blockIdx.y * blockDim.x + threadIdx.x; x < x1; x += gridDim.y * blockDim.x) row[x] = v;
    return;
  }
  uint4 vv = make_uint4(v, v, v, v);
  for (int x = xa + 4 * (blockIdx.y * blockDim.x + threadIdx.x); x < xb; x += 4 * gridDim.y * blockDim.x)
    *(uint4*)(row + x) = vv;
  if (blockIdx.y == 0) {
    for (int x = x0 + threadIdx.x; x < xa; x += blockDim.x) row[x] = v;
    for (int x = xb + threadIdx.x; x < x1; x += blockDim.x) row[x] = v;
  }
}

__global__ void wr_clear_rects_u8(const __grid_constant__ ClearRects p) {
  const int g = blockIdx.x, i = wr_clear_rect_of_row(p, g);
  const int4 r = p.r[i];
  uint8_t* row = p.base + (size_t)(r.y + (g - p.row0[i])) * p.pitch;
  for (int x = r.x + blockIdx.y * blockDim.x + threadIdx.x; x < r.z; x += gridDim.y * blockDim.x) row[x] = (uint8_t)p.v;
}
