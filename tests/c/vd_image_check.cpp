// Builds the view-conditioned decoder's weight image (nerf_from_image_b200/csrc/nfi_layout.h, the
// code the device runs) on the host: reads n_attention, scale1, scale3, pad and the fp32 weights
// w1 b1 w2 b2 w3 b3 from the file argv[1], writes the image's bytes to argv[2].
// tests/test_viewdir_weight_image.py un-permutes it.
#include <stdio.h>
#include <stdlib.h>

#include "nfi_layout.h"

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 3;
  float hdr[4];
  if (fread(hdr, 4, 4, f) != 4) return 4;
  const int A = (int)hdr[0], nl = A > 0 ? A : 3;
  const size_t n = 64 * 32 + 64 + 33 * 64 + 33 + (size_t)nl * 32 + nl;
  float* w = (float*)malloc(n * 4);
  if (fread(w, 4, n, f) != n) return 5;
  fclose(f);
  const float *w1 = w, *b1 = w1 + 64 * 32, *w2 = b1 + 64, *b2 = w2 + 33 * 64, *w3 = b2 + 33,
              *b3 = w3 + nl * 32;
  unsigned char* img = (unsigned char*)calloc(nfi::kVdBytes, 1);
  nfi::vd_weight_image_fill(w1, b1, w2, b2, w3, b3, A, img, hdr[1], hdr[2], hdr[3], 0, 1);
  FILE* o = fopen(argv[2], "wb");
  if (!o || fwrite(img, 1, nfi::kVdBytes, o) != (size_t)nfi::kVdBytes) return 6;
  fclose(o);
  return 0;
}
