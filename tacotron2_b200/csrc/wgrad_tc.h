// Tensor-core engine for the time-batched LSTM weight gradients of the decoder backward (wgrad_tc.cu).
#pragma once
#include "decoder.h"

namespace t2 {

struct WgJob {                          // one CTA: a 128 x 256 output tile of one K split
  const uint8_t* a; const uint8_t* b;   // first K chunk of the A (128 rows) and B (256 rows) operand images, [hi | lo] planes
  uint32_t a_stride, b_stride;          // bytes between consecutive K chunks
  int32_t nchunks;
  float* out; int32_t ldo;              // 128 x 256 fp32 tile, row-major
  const float* inv_scale;               // (128) per A row
};
constexpr int kWgTileA = 2 * 128 * 128, kWgTileB = 2 * 256 * 128;   // bytes of one A / B tile of one chunk
// The CTAs of a conv weight gradient (train_layers.cu), in launch order: tap k, A tile ia (128 output channels), B tile jb
// (256 input channels), K split sp (seg chunks of 64 padded rows).  A = G_z^T images (ntA tiles per chunk), B = the X^T
// images of tap k at img_b + k * b_img (ntB tiles per chunk); partial sums part (nsplit, coutP, ldp = 5 cinP).
struct WgConvJobs {
  const uint8_t* img_a; const uint8_t* img_b; size_t b_img;
  float* part; const float* inv;                 // inv: (coutP) per A row
  int nch, seg, nsplit, ntA, ntB, coutP, cinP, ldp;
  int count() const { return kConvK * ntA * ntB * nsplit; }
  __device__ WgJob operator()(int idx) const {
    const int sp = idx % nsplit; idx /= nsplit;
    const int jb = idx % ntB; idx /= ntB;
    const int ia = idx % ntA, k = idx / ntA;
    const int c0 = sp * seg;
    WgJob j;
    j.a_stride = (uint32_t)ntA * kWgTileA; j.b_stride = (uint32_t)ntB * kWgTileB;
    j.a = img_a + (size_t)c0 * j.a_stride + (size_t)ia * kWgTileA;
    j.b = img_b + (size_t)k * b_img + (size_t)c0 * j.b_stride + (size_t)jb * kWgTileB;
    j.nchunks = min(nch - c0, seg);
    j.out = part + ((size_t)sp * coutP + (size_t)ia * 128) * ldp + (size_t)k * cinP + (size_t)jb * 256;
    j.ldo = ldp;
    j.inv_scale = inv + ia * 128;
    return j;
  }
};
int wg_run_jobs(const WgConvJobs& jobs, cudaStream_t s);
// wg_colstats leaves its per-split partials in stat_ws: kWgStatSplit x [column max |x| (C) | column sum (C)]
constexpr int kWgStatSplit = 64;
size_t wg_colstats_ws_bytes(int C);
int wg_colstats(const float* x, long rows, int C, float* stat_ws, float* scale, float* inv_scale, float* colsum, cudaStream_t s);
int wg_transpose_images(const float* src, long ld, long row0, long rows_total, int chunk_rows, int nchunks, int C, int TR,
                        const float* scale, uint8_t* img, cudaStream_t s);

// K chunks of 64 batch rows per K split; a decoder step is ceil(B / 64) chunks, so `n` = T x ceil(B / 64)
constexpr int kWgSeg = 100;
inline int wgrad_seg(int n) { int seg = kWgSeg; while ((n + seg - 1) / seg > 15) seg += 50; return seg; }
struct WgradWs {                        // every region 1024-aligned
  uint8_t* img_a[2];                    // dG^T images of both LSTMs
  uint8_t *img_x2, *img_ctx, *img_ha, *img_hd;   // operand images (ctx sized like ha)
  float* part;                          // K-split partial sums of both LSTMs
  float *stat, *scale, *inv[2], *colsum;
};
void wgrad_tc_layout(Carve& c, int B, int T, WgradWs* w);
int wgrad_tc_run(T2Model* m, int B, int T, const float* dga, const float* dgd, const float* x2, const DecoderStash& st,
                 float* const* G, const WgradWs& w, cudaStream_t s);

}  // namespace t2
