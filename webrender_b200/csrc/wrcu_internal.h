// wrcu_internal.h — private definitions of the H100 frame-draw backend.
//
// Layout of the implementation (all sm_90a CUDA, no CPU fallback):
//   wrcu_api.cu      C ABI (include/wrcu.h): context, textures, frame tables,
//                    target binding, clears, draw dispatch.  What the draw
//                    path knows about each program kind (WRCU_KIND_*) is one
//                    row of its `kinds` table; wr_setup_batch picks the
//                    kind's set-up.
//   cmd.cuh          DrawCmd records produced by the per-kind "setup" kernels
//                    (= the reference's vertex stage, one thread per instance).
//   blend.cuh        The blend stage (bit-identical integer math to
//                    swgl/src/blend.h) as device functions.
//   raster.cuh       Tile-resident raster kernels: one CTA owns a 128x8-pixel
//                    framebuffer tile, keeps it in registers, walks the batch's
//                    commands IN ORDER, blends, and writes the tile once.
//   fold.cuh         Solid batches as per-channel lookup tables (wr_fold_solid).
//   setup_*.cuh      Vertex stages per BatchKind.
#pragma once

#ifdef WRCU_HOSTEMU
#include "hostemu_shim.h"  // tests only: g++ build of the device functions (symbols wremu_*)
#define WRD static inline
#define WRD_MEMBER static inline
#define WRD_METHOD inline
#define WRD_SHARED static inline
#else
#include <cuda_runtime.h>
#define WRD __device__ __forceinline__
#define WRD_MEMBER __device__ static __forceinline__
#define WRD_METHOD __device__ __forceinline__
// Large helpers every kernel uses (exact running sums, the blend stage, span partitions, sampling).  Measured
// both ways: as real functions (__noinline__, pixel loop rolled) the kernels are a third of the size and small
// batches run faster, but the 4K text / image / video passes lose more to call overhead and spilled row state —
// so they stay inlined.
#define WRD_SHARED __device__ __forceinline__
#endif
#include <stdint.h>
#include <utility>
#include <vector>
#include <stdio.h>
#include <string.h>

#include "../../include/wrcu.h"

#define WRCU_TILE_W 128
#define WRCU_TILE_H 8
#define WRCU_THREADS 256

struct WrTexture {
  int fmt = 0, w = 0, h = 0, bpp = 0, filter = WRCU_LINEAR;
  size_t pitch = 0;
  uint8_t* dptr = nullptr;
  bool live = false;
  bool imported = false;      // aliases another context's memory (wrcu_texture_import): never freed here
  bool ipc_mapped = false;    //   ... through cudaIpcOpenMemHandle (another process)
  bool has_tmap = false;      // a 2-D TMA tensor map of this texture sits in the context's device table
  int tmap_slot = 0;          //   ... in this slot
  uint64_t pending_read = 0;  // fence of an in-flight async readback of this texture
};

// Device-side view of a texture (passed by value to kernels).
struct TexView {
  const uint8_t* ptr;
  int w, h;
  int pitch;   // bytes
  int filter;  // WRCU_NEAREST / WRCU_LINEAR (already demoted if w < 2)
  int fmt;
  int tmap_id;  // index of this texture's TMA tensor map in the context's device table; 0 = none
};

// Device pointers to the per-frame data tables (16-byte texels).
struct FrameTablesDev {
  const float4* prim_headers_f; int n_prim_headers_f;
  const int4* prim_headers_i;   int n_prim_headers_i;
  const float4* transforms;     int n_transforms;
  const float4* render_tasks;   int n_render_tasks;
  const float4* gpu_cache;      int n_gpu_cache;
  const float4* gpu_buffer_f;   int n_gpu_buffer_f;
  const int4* gpu_buffer_i;     int n_gpu_buffer_i;
};

// Bound render target + the state draw_quad depends on
// (swgl/src/rasterize.h:1549-1632).
struct TargetDev {
  uint8_t* color;
  int color_pitch;
  int fmt;  // WRCU_FMT_RGBA8 | WRCU_FMT_R8
  int w, h;
  uint32_t* depth;  // nullptr when no depth test for this draw
  int depth_pitch;
  float proj[16];
  int vp[4];
  // scissor ∩ target bounds, as ints
  int cx0, cy0, cx1, cy1;
  int tmap_id;  // TMA tensor map of the colour target (0 = none)
};

// Bump arena: pinned host staging + device mirror, double-buffered per frame.
struct Arena {
  uint8_t* host = nullptr;
  uint8_t* dev = nullptr;
  size_t cap = 0, used = 0;
  cudaEvent_t done = nullptr;  // recorded at frame end
  bool in_flight = false;
};

struct wrcu_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  int sticky_error = 0;
  char err[512] = {0};
  static const int MAX_TEX = 8192;
  WrTexture tex[MAX_TEX];
  FrameTablesDev tables = {};
  // target
  wrcu_tex color_tex = 0, depth_tex = 0;
  float proj[16] = {0};
  int vp[4] = {0, 0, 0, 0};
  // arenas
  Arena arena[2];
  int cur_arena = 0;
  // scratch for commands
  void* cmd_hot = nullptr;
  void* cmd_cold = nullptr;
  int* batch_info = nullptr;  // ring of 4 BatchInfo records (bbox, flags)
  unsigned draw_seq = 0;
  // bitmask bins of the current batch (grown on demand)
  uint32_t* bin_mask = nullptr;
  size_t bin_cap_words = 0;
  int* dev_err = nullptr;     // count of instances rejected by setup kernels (sticky until read)
  size_t cmd_cap = 0;
  // stats / timing
  wrcu_stats stats = {};
  cudaEvent_t t0 = nullptr, t1 = nullptr;
  cudaEvent_t p0 = nullptr, p1 = nullptr;  // wrcu_profile_enable: around the last draw's raster kernels
  bool profile = false, profile_valid = false;
  int sm_count = 132;
  // asynchronous readback: second stream + a ring of fences
  static const int N_FENCES = 8;
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t ready_ev = nullptr;
  cudaEvent_t fence_ev[N_FENCES] = {};
  uint64_t fence_id[N_FENCES] = {};
  uint64_t next_fence = 1;
  // persistent GPU cache (wrcu_gpu_cache_update): rows of 1024 float4 blocks
  float4* gpu_cache_dev = nullptr;
  int gpu_cache_rows = 0;
  bool gpu_cache_bound = false;  // this frame's tables.gpu_cache is the persistent cache (not in an arena)
  std::vector<std::pair<uint8_t*, size_t>> host_allocs;  // wrcu_host_alloc blocks (staged without a copy)
  float* row_tab = nullptr;      // row-table pool of the current batch (CmdCold::row_off)
  int row_cap = 0;               // floats
  int flat_max = 2;          // solid batches of <= flat_max layers take the streaming kernel
  int fold_min = 0;          // solid batches of >= fold_min layers get lookup tables (wr_fold_solid) for full-cover tiles
  uint8_t* fold_lut = nullptr;  // those tables (WR_FOLD_SLOT bytes per BatchInfo record), indexed like batch_info
  int fast_ctas_per_sm = 0;  // resident CTAs/SM of the solid-premult kernel (occupancy API)
  // TMA: one 128-byte CUtensorMap per RGBA8 texture (box 256x16 px), built on the host at texture
  // creation (cuTensorMapEncodeTiled through cudaGetDriverEntryPoint) and kept in a device table
  // multi-GPU flags (wrcu_peer_*): own flag words + mapped peers
  uint32_t* flags = nullptr;
  int n_flags = 0;
  struct PeerFlags { uint32_t* ptr; int count; bool ipc; };
  std::vector<PeerFlags> peers;
  // deferred submission (wrcu_api.cu: PendingOp, flush_pending): clears and batches queue up; one H2D copy, ONE
  // set-up launch for all queued batches, then the clears / raster launches in order
  static const int QMAX = 1024;
  void* pending_ops = nullptr;   // std::vector<PendingOp>*
  size_t pend_instances = 0;
  bool in_flush = false;
  // side streams of a submission (flush_multi_stream): one per render target, round robin (WRCU_STREAMS, 1 = off)
  int n_streams = 8;
  bool side_reduce = false;      // set while a submission with >= 4 render targets is being launched
  int side_ctas_per_sm = 1;      // persistent CTAs per SM of a small batch's raster kernel on a side stream (WRCU_SIDE_CTAS)
  std::vector<cudaStream_t> side;
  std::vector<cudaEvent_t> op_events, join_ev;
  bool plain_next = false;         // the next chained launch follows an event wait: launch it the ordinary way
  bool early_clear = true;         // clears wait for the fork point BEFORE the set-up launch (WRCU_EARLY_CLEAR=0: after it)
  int glyph_ctas = 6;              // persistent CTAs per SM of the glyph-major kernel (WRCU_GLYPH_CTAS)
  bool strip = true;               // strip mode of the tile kernel for wide single-surface batches (WRCU_STRIP=0: off)
  bool yuv_wide = false;           // composite YUV through the one-CTA-per-SM variant (WRCU_YUV_WIDE=1)
  bool glyph_major = true;         // text batches go through wr_raster_glyphs first (WRCU_GLYPH_MAJOR=0: tile kernel only)
  cudaEvent_t fork_ev = nullptr;
  cudaEvent_t fork0_ev = nullptr;  // recorded before the submission's H2D copy: leading clears wait only for this
  cudaStream_t launch_stream = nullptr;  // where launch_clear / launch_raster queue (the context's stream, or a side stream)
  bool pdl = true;               // raster launches chained with programmatic stream serialization (WRCU_PDL=0: off)
  bool immediate = false;        // WRCU_IMMEDIATE=1: flush after every call (A/B measurements)
  int flush_parity = 0;          // which half of batch_info / pool_ctr the current submission uses
  int* pool_ctr = nullptr;       // 2 x {row-table floats, depth-run words} handed out (device)
  size_t dirty_lo = 0, dirty_hi = 0;  // arena range staged on the host but not yet copied to the device
  int n_wait_kernel = 0, n_wait_event = 0;  // wrcu_peer_wait: polling kernels / event waits queued (diagnostics)
  uint32_t* fail_pool = nullptr;  // depth-run bitmaps of the current batch (CmdCold::fail_off)
  int fail_cap = 0;               // words
  void* tmaps_dev = nullptr;
  static const int TMAP_SLOTS = 65536;  // 8 MiB of 128-byte records; slot 0 = none
  int tmap_next = 1;
  bool tmap_wrapped = false;     // slots are being reused: kernels acquire the maps they use
  void* tmap_encode = nullptr;
  bool copy_attr_set = false;
};

int wrcu_fail(wrcu_ctx* c, int code, const char* fmt, ...);

#define WRCU_CUDA(c, call)                                                     \
  do {                                                                         \
    cudaError_t e_ = (call);                                                   \
    if (e_ != cudaSuccess)                                                     \
      return wrcu_fail((c), e_ == cudaErrorMemoryAllocation ? WRCU_ERR_OOM     \
                                                            : WRCU_ERR_CUDA,   \
                       "%s failed: %s", #call, cudaGetErrorString(e_));        \
  } while (0)
