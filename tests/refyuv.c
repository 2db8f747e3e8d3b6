/*
 * tests/refyuv.c -- TEST INFRASTRUCTURE (not product code).
 *
 * An application of the TurboJPEG YUV API: tj3EncodeYUV8 with row alignments 1, 4 and 64, and tj3EncodeYUVPlanes8
 * with explicit strides into buffers prefilled with 0xEE, for several subsamplings and pixel formats of one seeded
 * 97x61 image.  Every whole buffer (padding included) is written to <outdir>/<name>.bin, so a run in front of the
 * reference library and a run under the interposer can be compared file by file.  tests/test_yuv.py compiles it
 * against oracle/_ref/libturbojpeg_ref.so.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <turbojpeg.h>

static int dump(const char *dir, const char *name, const unsigned char *buf, size_t n)
{
  char path[1024];
  snprintf(path, sizeof path, "%s/%s.bin", dir, name);
  FILE *f = fopen(path, "wb");
  if (!f || fwrite(buf, 1, n, f) != n) { fprintf(stderr, "cannot write %s\n", path); return -1; }
  fclose(f);
  return 0;
}

int main(int argc, char **argv)
{
  if (argc != 2) { fprintf(stderr, "usage: refyuv outdir\n"); return 2; }
  const int w = 97, h = 61;
  const int samps[] = {TJSAMP_420, TJSAMP_422, TJSAMP_444, TJSAMP_GRAY, TJSAMP_440, TJSAMP_411, TJSAMP_441};
  const int pfs[] = {TJPF_RGB, TJPF_BGRX, TJPF_XRGB, TJPF_GRAY};
  unsigned int seed = 12345;
  unsigned char *src = malloc((size_t)w * h * 4);
  for (int i = 0; i < w * h * 4; i++) { seed = seed * 1103515245u + 12345u; src[i] = (unsigned char)(seed >> 16); }
  tjhandle tj = tj3Init(TJINIT_COMPRESS);
  if (!tj) return 1;
  for (unsigned s = 0; s < sizeof samps / sizeof *samps; s++)
    for (unsigned f = 0; f < sizeof pfs / sizeof *pfs; f++) {
      const int ss = samps[s], pf = pfs[f];
      if (pf == TJPF_GRAY && ss != TJSAMP_GRAY) continue;
      tj3Set(tj, TJPARAM_SUBSAMP, ss);
      char name[128];
      const int aligns[] = {1, 4, 64};
      for (int a = 0; a < 3; a++) {
        const size_t n = tj3YUVBufSize(w, aligns[a], h, ss);
        unsigned char *buf = malloc(n);
        memset(buf, 0xEE, n);
        if (tj3EncodeYUV8(tj, src, w, 0, h, pf, buf, aligns[a]) != 0) { fprintf(stderr, "tj3EncodeYUV8: %s\n", tj3GetErrorStr(tj)); return 1; }
        snprintf(name, sizeof name, "yuv8_s%d_pf%d_a%d", ss, pf, aligns[a]);
        if (dump(argv[1], name, buf, n)) return 1;
        free(buf);
      }
      /* explicit strides, and a source pitch wider than a row */
      const int np = ss == TJSAMP_GRAY ? 1 : 3, ps = tjPixelSize[pf];
      unsigned char *planes[3] = {NULL, NULL, NULL};
      int strides[3] = {0, 0, 0};
      size_t sizes[3] = {0, 0, 0};
      for (int c = 0; c < np; c++) {
        strides[c] = tj3YUVPlaneWidth(c, w, ss) + 5 + 3 * c;
        sizes[c] = (size_t)strides[c] * tj3YUVPlaneHeight(c, h, ss);
        planes[c] = malloc(sizes[c]);
        memset(planes[c], 0xEE, sizes[c]);
      }
      const int pitch = w * ps + 3;
      unsigned char *wide = malloc((size_t)pitch * h);
      for (int y = 0; y < h; y++) memcpy(wide + (size_t)y * pitch, src + (size_t)y * w * ps, (size_t)w * ps);
      if (tj3EncodeYUVPlanes8(tj, wide, w, pitch, h, pf, planes, strides) != 0) { fprintf(stderr, "tj3EncodeYUVPlanes8: %s\n", tj3GetErrorStr(tj)); return 1; }
      for (int c = 0; c < np; c++) {
        snprintf(name, sizeof name, "planes_s%d_pf%d_c%d", ss, pf, c);
        if (dump(argv[1], name, planes[c], sizes[c])) return 1;
        free(planes[c]);
      }
      free(wide);
    }
  tj3Destroy(tj);
  free(src);
  return 0;
}
