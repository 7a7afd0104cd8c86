// wgrad_items.cuh -- the weight-gradient work list of the SIMT wgrad kernel:
// one item per (gemm layer, output-row block, input-column block) + one per narrow head.
#pragma once
#include "common.cuh"

namespace nerfb200 {

struct WgItem {
  int kind;      // 0: gemm weight block with X from the stash, 1: X = encoding, 2: head
  int t;         // gemm index (kind 0/1) or head index (kind 2)
  int n0, nblk;  // output-row block
  int k0, kblk;  // input-column block (kind 0: offset in the h part; kind 1: padded-to-16 encoding width)
  int bias;      // this item also reduces the bias gradient
};

__host__ __device__ inline int wg_item_count(const Plan& p) {
  int n = 0;
  for (int t = 0; t < p.n_gemm; ++t) {
    const int nb = p.g[t].n / 128 > 0 ? (p.g[t].n + 127) / 128 : 1;
    const int kb = (p.g[t].k_h + 127) / 128;
    n += nb * (kb + (p.g[t].k_enc > 0 ? 1 : 0));
  }
  return n + p.n_head;
}

__host__ __device__ inline int wg_imin(int a, int b) { return a < b ? a : b; }

__host__ __device__ inline WgItem wg_decode(const Plan& p, int item) {
  WgItem it;
  for (int t = 0; t < p.n_gemm; ++t) {
    const GemmLayer& g = p.g[t];
    const int nb = (g.n + 127) / 128;
    const int kb = (g.k_h + 127) / 128;
    const int per = kb + (g.k_enc > 0 ? 1 : 0);
    if (item < nb * per) {
      const int bn = item / per, bk = item - bn * per;
      it.t = t;
      it.n0 = bn * 128;
      it.nblk = wg_imin(128, g.n - it.n0);
      if (bk < kb) {
        it.kind = 0;
        it.k0 = bk * 128;
        it.kblk = wg_imin(128, g.k_h - it.k0);
        it.bias = (bk == 0);
      } else {
        it.kind = 1;
        it.k0 = 0;
        it.kblk = (g.enc_real + 15) & ~15;
        it.bias = (kb == 0);
      }
      return it;
    }
    item -= nb * per;
  }
  it.kind = 2;
  it.t = item;
  it.n0 = 0; it.nblk = p.h[item].n_out; it.k0 = 0; it.kblk = p.h[item].k; it.bias = 1;
  return it;
}

}  // namespace nerfb200
