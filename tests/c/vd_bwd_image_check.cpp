// Builds the view-conditioned decoder's backward weight image (nerf_from_image_b200/csrc/
// nfi_layout.h, vd_bwd_weight_image_fill: the code the device runs) on the host: reads n_attention
// and the fp32 weights w1 [64 x 32], w2 [33 x 64], w3 [A or 3 x 32] from the file argv[1], writes
// the image's bytes to argv[2].  tests/test_viewdir_backward_image.py un-permutes it.
#include <stdio.h>
#include <stdlib.h>

#include "nfi_layout.h"

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 3;
  float hdr[1];
  if (fread(hdr, 4, 1, f) != 1) return 4;
  const int A = (int)hdr[0], nl = A > 0 ? A : 3;
  const size_t n = 64 * 32 + 33 * 64 + (size_t)nl * 32;
  float* w = (float*)malloc(n * 4);
  if (fread(w, 4, n, f) != n) return 5;
  fclose(f);
  const float *w1 = w, *w2 = w1 + 64 * 32, *w3 = w2 + 33 * 64;
  unsigned char* img = (unsigned char*)calloc(nfi::kVbBytes, 1);
  nfi::vd_bwd_weight_image_fill(w1, w2, w3, A, img, 0, 1);
  FILE* o = fopen(argv[2], "wb");
  if (!o || fwrite(img, 1, nfi::kVbBytes, o) != (size_t)nfi::kVbBytes) return 6;
  fclose(o);
  return 0;
}
