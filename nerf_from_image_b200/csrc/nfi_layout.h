// Operand layouts of the tensor-core kernels as plain index arithmetic, compilable by a host
// C++ compiler without the CUDA toolkit (tests/c/vd_image_check.cpp runs them on the CPU):
// the SWIZZLE_128B tile offset, the K permutation of a register A fragment, and the weight images
// of the view-direction-conditioned kernels (render_forward_pipe / render_backward_pipe<...,
// VD = true>; tests/c/vd_bwd_image_check.cpp runs the backward one).
#pragma once
#include <stdint.h>
#include <string.h>

#ifdef __CUDACC__
#define NFI_HD __host__ __device__ __forceinline__
#else
#define NFI_HD inline
#endif

namespace nfi {
namespace tc {

// byte offset of (row, 16-byte chunk) inside a [rows x 128 B] SWIZZLE_128B tile
NFI_HD uint32_t sw128_offset(int row, int chunk) {
  return (uint32_t)((row >> 3) * 1024 + (row & 7) * 128 + ((chunk ^ (row & 7)) << 4));
}

// K position, inside its block of 8, at which a register A fragment holds hidden unit j (see
// nfi_tc.cuh): units 2t and 2t + 1 of the block sit at positions t and t + 4
NFI_HD constexpr int kpos_of_hidden(int j) {
  return (j & ~7) | ((j & 1) ? 4 + ((j >> 1) & 3) : ((j >> 1) & 3));
}
// accumulator register e of a column block (rows g / g + 8, columns 2t / 2t + 1) -> A-fragment
// register of the same element: a0 = (g, t), a1 = (g + 8, t), a2 = (g, t + 4), a3 = (g + 8, t + 4)
NFI_HD constexpr int afrag_slot(int e) { return ((e & 1) << 1) | (e >> 1); }

}  // namespace tc

// decoder outputs: the distance and A colour logits (three when A = 0), padded for the kernels
constexpr int nout_of(int n_attention) { return 1 + (n_attention > 0 ? n_attention : 3); }
constexpr int nout_pad_of(int n_attention) {
  return nout_of(n_attention) <= 4 ? 4 : (nout_of(n_attention) <= 12 ? 12 : 16);
}

// ---------------------------------------------------------------------------
// Workspace of the render kernels (bytes from params.workspace).
//   forward   [0, kFwdImageSlot): the weight image (kVdFwdImageSlot with a view), then the
//             scratch slabs of the coarse samples, then, when render_normals_pipe runs, its
//             backward weight image (kBwdImageBytes; nfi_render.cu computes the offsets)
//   backward  the forward image at 0, the backward image at kBwdImageOffset, then from
//             kWgAccOffset render_wgrad_pipe's accumulator rows, one per CTA of at most
//             kMaxPersistentCtas (NFI_BACKWARD_WORKSPACE_BYTES); with a view both images take
//             48 KiB slots (kVdBwdImageOffset below, NFI_VIEW_BACKWARD_WORKSPACE_BYTES)
// ---------------------------------------------------------------------------
constexpr int kFwdImageSlot = 32768;    // nfi::kWiBytes rounded up
constexpr int kVdFwdImageSlot = 65536;  // kVdBytes rounded up
constexpr int kBwdImageOffset = 32768;
constexpr int kBwdImageBytes = 32768;   // nfi::kWbBytes
constexpr int kWgAccOffset = kBwdImageOffset + kBwdImageBytes;
constexpr size_t kWgAccBytesPerCta = 128 * 64 * sizeof(float);
constexpr size_t kMaxPersistentCtas = 160;  // >= SM count of any sm_90 part (H100 SXM: 132)

// ---------------------------------------------------------------------------
// Weight image of the view-direction-conditioned decoder (models/generator.py:189-253,662-663):
//   layer 1   W1 [64 x 32], b1                       as in the plain image (nfi_forward_tc.cuh)
//   layer 2   W2 [33 x 64]: row 0 = distance, rows 1..32 = features.  Stored as a [40 x 64] B
//             operand whose output column c < 32 is feature c (w2 row c + 1) and column 32 the
//             distance (w2 row 0); columns 33..39 are zero.  K positions in fragment order.
//   layer 3   W3 [A or 3 x 32] as a [16 x 32] B operand: output column 0 has zero weights (the
//             distance is moved there in registers), column 1 + a is w3 row a; K position of
//             feature c = kpos_of_hidden(c), the layer-2 accumulator being layer 3's A fragment.
//   biases    b1 [64]; b2f [32] = b2[1..32] (added to the features with the ray's view features);
//             head [16] = what the shading warpgroup adds to a D2 row: b2[0], then b3, then the
//             padding value of the unused logits.
// `scale1` multiplies W1 / b1, `scale3` W3 / b3 (the colour logits), `pad` fills head[1 + A ..].
// ---------------------------------------------------------------------------
constexpr int kVdW2Cols = 40;                      // layer-2 output columns (N of the wgmma)
constexpr int kVdW2KBlockBytes = kVdW2Cols * 128;  // one [40 x 32] SWIZZLE_128B K-block
constexpr int kVdW1Hi = 0;                         // [64 x 32] SW128, 8 KB
constexpr int kVdW1Lo = 8192;
constexpr int kVdW2Hi = 16384;                     // two K-blocks, 10 KB
constexpr int kVdW2Lo = kVdW2Hi + 2 * kVdW2KBlockBytes;
constexpr int kVdW3Hi = kVdW2Lo + 2 * kVdW2KBlockBytes;  // [16 x 32] SW128, 2 KB
constexpr int kVdW3Lo = kVdW3Hi + 2048;
constexpr int kVdB1 = kVdW3Lo + 2048;              // 64 floats
constexpr int kVdB2f = kVdB1 + 256;                // 32 floats
constexpr int kVdHead = kVdB2f + 128;              // 16 floats
constexpr int kVdBytes = kVdHead + 64;             // 41408
static_assert(kVdW3Hi % 1024 == 0 && kVdBytes % 16 == 0, "SWIZZLE_128B atoms / bulk-copy size");
static_assert(kVdBytes <= kVdFwdImageSlot, "weight image larger than the workspace header");

// output column of layer 2 that holds row `row` of w2
NFI_HD constexpr int vd_w2_col(int row) { return row == 0 ? 32 : row - 1; }
// byte offset, inside a W2 hi / lo block, of (output column, hidden unit j)
NFI_HD uint32_t vd_w2_offset(int col, int j) {
  const int jp = tc::kpos_of_hidden(j);
  return (uint32_t)((jp >> 5) * kVdW2KBlockBytes) + tc::sw128_offset(col, (jp & 31) >> 2) +
         (uint32_t)(jp & 3) * 4u;
}
// byte offset, inside a W3 hi / lo block, of (output column, feature c)
NFI_HD uint32_t vd_w3_offset(int col, int c) {
  const int cp = tc::kpos_of_hidden(c);
  return tc::sw128_offset(col, cp >> 2) + (uint32_t)(cp & 3) * 4u;
}

// x with the low 13 mantissa bits cleared: exactly representable in TF32
NFI_HD float vd_tf32_hi(float x) {
  uint32_t u;
  memcpy(&u, &x, 4);
  u &= 0xFFFFE000u;
  memcpy(&x, &u, 4);
  return x;
}
NFI_HD void vd_put_split(unsigned char* img, int hi_base, int lo_base, uint32_t off, float w) {
  const float hi = vd_tf32_hi(w);
  const float lo = w - hi;
  memcpy(img + hi_base + off, &hi, 4);
  memcpy(img + lo_base + off, &lo, 4);
}

// Worker `idx` of `n` fills its share of the image (a CUDA block's threads, or 0 of 1 on the host).
NFI_HD void vd_weight_image_fill(const float* w1, const float* b1, const float* w2, const float* b2,
                                 const float* w3, const float* b3, int n_attention,
                                 unsigned char* img, float scale1, float scale3, float pad,
                                 int idx, int n) {
  const int nlogit = n_attention > 0 ? n_attention : 3;
  for (int i = idx; i < 64 * 32; i += n) {
    const int j = i / 32, k = i % 32;  // W1[j][k]
    vd_put_split(img, kVdW1Hi, kVdW1Lo, tc::sw128_offset(j, k >> 2) + (uint32_t)(k & 3) * 4u,
                 w1[i] * scale1);
  }
  for (int i = idx; i < kVdW2Cols * 64; i += n) {
    const int col = i / 64, j = i % 64;
    const float w = col < 32 ? w2[(col + 1) * 64 + j] : (col == 32 ? w2[j] : 0.f);
    vd_put_split(img, kVdW2Hi, kVdW2Lo, vd_w2_offset(col, j), w);
  }
  for (int i = idx; i < 16 * 32; i += n) {
    const int col = i / 32, c = i % 32;
    const float w = (col >= 1 && col <= nlogit) ? w3[(col - 1) * 32 + c] * scale3 : 0.f;
    vd_put_split(img, kVdW3Hi, kVdW3Lo, vd_w3_offset(col, c), w);
  }
  float* b1i = reinterpret_cast<float*>(img + kVdB1);
  float* b2f = reinterpret_cast<float*>(img + kVdB2f);
  float* head = reinterpret_cast<float*>(img + kVdHead);
  for (int i = idx; i < 64; i += n) b1i[i] = b1[i] * scale1;
  for (int i = idx; i < 32; i += n) b2f[i] = b2[1 + i];
  for (int i = idx; i < 16; i += n)
    head[i] = i == 0 ? b2[0] : (i <= nlogit ? b3[i - 1] * scale3 : pad);
}

// ---------------------------------------------------------------------------
// Backward weight image of the view-conditioned decoder (render_backward_pipe<..., VD = true>),
// loaded beside the forward image above.  All weights in natural units (no log2 e): the shading
// warpgroup's dOut is the derivative with respect to the natural-units outputs.
//   W1^T / 3  [32 rows = channel c][64 K = hidden j] as two [32 x 32] K-blocks (4 KB each), K
//             positions in fragment order: D4 = dpre (W1 / 3), dpre a register A fragment
//   W2f^T     [64 rows = hidden j][32 K = feature c], K in fragment order: D3 = dF W2[1..32],
//             dF (the layer-3 reverse accumulator) a register A fragment
//   W3^T      [32 rows = feature c][32 K = output o, 16 used]: dG = dOut W3, dOut loaded from
//             shared memory in natural K order; K position 0 (the distance) has zero weights,
//             K position 1 + a is w3 row a
//   w2d       w2 row 0 (the distance row) in fp32: its part of D3, dDist w2d, is added on the
//             CUDA cores
// Each operand block is a multiple of 1 KB (SWIZZLE_128B atoms); hi / lo TF32 parts.
// ---------------------------------------------------------------------------
constexpr int kVbW1tHi = 0;
constexpr int kVbW1tLo = 8192;
constexpr int kVbW2tHi = 16384;  // [64 x 32] SW128, 8 KB
constexpr int kVbW2tLo = 24576;
constexpr int kVbW3Hi = 32768;   // [32 x 32] SW128, 4 KB
constexpr int kVbW3Lo = 36864;
constexpr int kVbW2d = 40960;    // 64 floats
constexpr int kVbBytes = kVbW2d + 256;  // 41216
static_assert(kVbBytes % 16 == 0, "bulk-copy size");
// the backward's workspace: forward image in [0, 48 KiB), backward image in [48 KiB, 96 KiB)
// (NFI_VIEW_BACKWARD_WORKSPACE_BYTES)
constexpr int kVdBwdImageOffset = 49152;
constexpr int kVdBackwardWorkspaceBytes = 2 * kVdBwdImageOffset;
static_assert(kVdBytes <= kVdBwdImageOffset && kVbBytes <= kVdBwdImageOffset,
              "a weight image overflows its workspace slot");

// byte offset, inside a W1^T / 3 hi / lo block, of (channel c, hidden unit j)
NFI_HD uint32_t vb_w1t_offset(int c, int j) {
  const int jp = tc::kpos_of_hidden(j);
  return (uint32_t)((jp >> 5) * 4096) + tc::sw128_offset(c, (jp & 31) >> 2) +
         (uint32_t)(jp & 3) * 4u;
}
// byte offset, inside a W2f^T hi / lo block, of (hidden unit j, feature c)
NFI_HD uint32_t vb_w2t_offset(int j, int c) {
  const int cp = tc::kpos_of_hidden(c);
  return tc::sw128_offset(j, cp >> 2) + (uint32_t)(cp & 3) * 4u;
}
// byte offset, inside a W3^T hi / lo block, of (feature c, output o)
NFI_HD uint32_t vb_w3t_offset(int c, int o) {
  return tc::sw128_offset(c, o >> 2) + (uint32_t)(o & 3) * 4u;
}

// Worker `idx` of `n` fills its share of the backward image (w2 [33 x 64], w3 [A or 3 x 32]).
NFI_HD void vd_bwd_weight_image_fill(const float* w1, const float* w2, const float* w3,
                                     int n_attention, unsigned char* img, int idx, int n) {
  const int nlogit = n_attention > 0 ? n_attention : 3;
  for (int i = idx; i < 32 * 64; i += n) {
    const int c = i / 64, j = i % 64;
    vd_put_split(img, kVbW1tHi, kVbW1tLo, vb_w1t_offset(c, j), w1[j * 32 + c] * (1.f / 3.f));
  }
  for (int i = idx; i < 64 * 32; i += n) {
    const int j = i / 32, c = i % 32;
    vd_put_split(img, kVbW2tHi, kVbW2tLo, vb_w2t_offset(j, c), w2[(c + 1) * 64 + j]);
  }
  for (int i = idx; i < 32 * 32; i += n) {
    const int c = i / 32, o = i % 32;
    const float w = (o >= 1 && o <= nlogit) ? w3[(o - 1) * 32 + c] : 0.f;
    vd_put_split(img, kVbW3Hi, kVbW3Lo, vb_w3t_offset(c, o), w);
  }
  float* w2d = reinterpret_cast<float*>(img + kVbW2d);
  for (int i = idx; i < 64; i += n) w2d[i] = w2[i];
}

}  // namespace nfi
