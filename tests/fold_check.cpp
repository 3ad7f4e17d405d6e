// The lookup tables of a solid batch (csrc/fold.cuh, wr_fold_host: the device fold step by step) against
// sequential blending: seeded random stacks of 1 .. 1000 layers, valid and over-range colours, alpha 0 and 255
// included, some commands empty; every input of every channel must match.
#include <stdio.h>
#include <stdint.h>
#include <vector>
#define WRCU_HOSTEMU 1
#include "../webrender_b200/csrc/fold.cuh"

static uint32_t rng_state = 2463534242u;
static uint32_t rnd() { rng_state ^= rng_state << 13; rng_state ^= rng_state >> 17; rng_state ^= rng_state << 5; return rng_state; }

// premultiplied over as the reference writes it (blend.h:473-474): sat(src + dst - muldiv255(dst, src.a))
static int over(int d, int s, int a) {
  const int v = s + d - ((d * a + d) >> 8);
  return v > 255 ? 255 : v;
}

int main() {
  long bad = 0, stacks = 0;
  std::vector<int> sizes;
  for (int n = 1; n <= 40; n++) sizes.push_back(n);
  for (int n : {63, 64, 65, 127, 128, 129, 255, 256, 257, 999, 1000}) sizes.push_back(n);
  for (int i = 0; i < 60; i++) sizes.push_back(1 + (int)(rnd() % 1000));
  for (int n : sizes) {
    for (int mode = 0; mode < 3; mode++) {  // 0: valid colours, 1: over-range colours, 2: valid colours, saturating path
      std::vector<CmdHot> hot((size_t)n);
      bool valid = true;
      for (int i = 0; i < n; i++) {
        CmdHot& c = hot[(size_t)i];
        memset(&c, 0, sizeof c);
        const bool empty = rnd() % 16 == 0;
        c.x0 = 0; c.y0 = 0; c.x1 = empty ? 0 : 64; c.y1 = empty ? 0 : 8;
        const uint32_t r = rnd() % 8;
        const int a = r == 0 ? 0 : r == 1 ? 255 : (int)(rnd() % 256);
        c.col[3] = (uint16_t)a;
        for (int ch = 0; ch < 3; ch++) c.col[ch] = (uint16_t)(mode == 1 ? rnd() % 256 : (a ? rnd() % (a + 1) : 0));
        if (!empty && (c.col[0] > a || c.col[1] > a || c.col[2] > a)) valid = false;
      }
      uint8_t tab[WR_FOLD_ENTRIES];
      wr_fold_host(hot.data(), n, mode != 2 && valid, tab);
      stacks++;
      for (int ch = 0; ch < 4; ch++)
        for (int v = 0; v < 256; v++) {
          int d = v;
          for (const CmdHot& c : hot)
            if (c.x1 > c.x0) d = over(d, c.col[ch], c.col[3]);
          if (tab[ch * 256 + v] != d) {
            if (bad < 10) printf("MISMATCH n=%d mode=%d ch=%d v=%d table=%d sequential=%d\n", n, mode, ch, v, tab[ch * 256 + v], d);
            bad++;
          }
        }
    }
  }
  printf("stacks %ld bad %ld\n", stacks, bad);
  return bad != 0;
}
