// clear_rects.cuh — the launch parameters of the rect-list clear (wrcu_clear_rects).
//
// Up to WR_CLEAR_RECTS_MAX clamped, non-empty rects of one target are cleared in one launch.  The rects
// travel by value in the launch parameters, so the op reads nothing the submission's host-to-device copy
// writes and can start ahead of it like any clear.  The rows of all rects are numbered one after another
// (row0 = each rect's first row); CTA (x = row, y = column slice) writes one row the way wr_clear_u32 /
// wr_clear_u8 write a row of one rect.
#pragma once
#include <stdint.h>

#define WR_CLEAR_RECTS_MAX 64
struct ClearRects {
  uint8_t* base;
  int pitch, n;
  uint32_t v;
  int4 r[WR_CLEAR_RECTS_MAX];        // x0, y0, x1, y1
  int row0[WR_CLEAR_RECTS_MAX + 1];  // row0[n] = rows in all
};

#ifndef WRCU_HOSTEMU
__global__ void wr_clear_rects_u32(const __grid_constant__ ClearRects p);
__global__ void wr_clear_rects_u8(const __grid_constant__ ClearRects p);
#endif
