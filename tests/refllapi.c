/*
 * tests/refllapi.c -- TEST INFRASTRUCTURE (not product code).
 *
 * An application of the lossless encoder through the libjpeg and TurboJPEG APIs.  It prints, on stdout, everything an
 * application can see of each encode: a hash of the file, every progress-monitor call, and the fields of the object
 * that jpeg_start_compress changes in lossless mode.  tests/test_lossless_api.py compiles it against the reference
 * library (oracle/_ref) and runs it with and without the interposer; the two outputs must be identical.
 *
 *   tj3Compress8/12/16 with TJPARAM_LOSSLESS, TJPARAM_LOSSLESSPSV, TJPARAM_LOSSLESSPT and TJPARAM_RESTARTROWS;
 *   libjpeg objects at 8, 12 and 16 bits with a progress monitor; an object that asked for raw data before
 *   jpeg_enable_lossless and then writes scanlines; the overrides of colour space, sampling and smoothing; a hand-made
 *   two-scan lossless script; a progressive script over jpeg_enable_lossless (a lossy object).
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <setjmp.h>
#define JPEG_INTERNALS
#include "jinclude.h"
#include "jpeglib.h"
#include <turbojpeg.h>

#define W 37
#define H 23

struct err_mgr { struct jpeg_error_mgr pub; jmp_buf jb; };
static void on_error(j_common_ptr c)
{
  char msg[JMSG_LENGTH_MAX];
  (*c->err->format_message)(c, msg);
  printf("  error: %s\n", msg);
  longjmp(((struct err_mgr *)c->err)->jb, 1);
}
static void on_message(j_common_ptr c, int lvl) { (void)c; (void)lvl; }

static void on_progress(j_common_ptr c)
{
  printf("  progress %d %d %ld %ld\n", c->progress->completed_passes, c->progress->total_passes, c->progress->pass_counter, c->progress->pass_limit);
}

static unsigned long long fnv(const unsigned char *d, unsigned long n)
{
  unsigned long long h = 14695981039346656037ull;
  for (unsigned long i = 0; i < n; i++) { h ^= d[i]; h *= 1099511628211ull; }
  return h;
}

/* seeded samples below 1 << prec: a ramp plus noise, so that the predictors have something to do */
static void fill(unsigned short *s, int n, int nc, int prec, unsigned seed)
{
  for (int i = 0; i < n * nc; i++) {
    seed = seed * 1103515245u + 12345u;
    s[i] = (unsigned short)((i / nc % W * 5 + i / nc / W * 3) * ((1 << prec) / 256) + (seed >> 16) % 7) & ((1 << prec) - 1);
  }
}

static void print_state(j_compress_ptr c)
{
  printf("  lossless %d jpeg_color_space %d num_components %d", c->master->lossless, c->jpeg_color_space, c->num_components);
  for (int ci = 0; ci < c->num_components; ci++) {
    jpeg_component_info *k = &c->comp_info[ci];
    printf(" [%dx%d %ux%u du %d]", k->h_samp_factor, k->v_samp_factor, k->width_in_blocks, k->height_in_blocks, k->DCT_scaled_size);
  }
  printf(" total_iMCU_rows %u smoothing %d optimize %d raw_data_in %d global_state %d\n", c->total_iMCU_rows, c->smoothing_factor,
         c->optimize_coding, c->raw_data_in, c->global_state);
}

enum { PLAIN, RAW_FIRST, OVERRIDES, SCRIPT, PROGRESSIVE };

/* one libjpeg-API object: input_components samples per pixel of in_cs at prec bits, rows written `step` at a time */
static void api_encode(const char *name, int prec, J_COLOR_SPACE in_cs, int nc, int psv, int pt, int restart_rows, int variant, int step)
{
  struct jpeg_compress_struct c;
  struct err_mgr e;
  struct jpeg_progress_mgr prog;
  unsigned char *out = NULL;
  unsigned long outsize = 0;
  static jpeg_scan_info script[2];
  unsigned short *pix = malloc(sizeof(unsigned short) * W * H * nc);
  unsigned char *pix8 = malloc((size_t)W * H * nc);
  fill(pix, W * H, nc, prec, (unsigned)(prec * 131 + psv * 7 + variant));
  for (int i = 0; i < W * H * nc; i++) pix8[i] = (unsigned char)pix[i];
  printf("%s\n", name);
  c.err = jpeg_std_error(&e.pub);
  e.pub.error_exit = on_error; e.pub.emit_message = on_message;
  if (setjmp(e.jb)) { jpeg_destroy_compress(&c); free(out); free(pix); free(pix8); return; }
  jpeg_create_compress(&c);
  prog.progress_monitor = on_progress;
  /* the lossy device path reports each of its later passes in one call rather than row by row: only lossless objects
   * get a monitor here */
  c.progress = variant == PROGRESSIVE ? NULL : &prog;
  c.in_color_space = in_cs; c.input_components = nc;
  c.image_width = W; c.image_height = H;
  c.data_precision = prec;
  jpeg_c_set_int_param(&c, JINT_COMPRESS_PROFILE, JCP_FASTEST);
  jpeg_set_defaults(&c);
  c.restart_in_rows = restart_rows;
  if (variant == RAW_FIRST) c.raw_data_in = TRUE;
  if (variant == OVERRIDES) {
    jpeg_set_colorspace(&c, JCS_GRAYSCALE);
    c.comp_info[0].h_samp_factor = c.comp_info[0].v_samp_factor = 2;
    c.smoothing_factor = 30;
    c.optimize_coding = FALSE;
  }
  if (variant == PROGRESSIVE) jpeg_simple_progression(&c);
  if (variant == SCRIPT) {
    script[0].comps_in_scan = 2; script[0].component_index[0] = 0; script[0].component_index[1] = 2;
    script[0].Ss = psv; script[0].Se = 0; script[0].Ah = 0; script[0].Al = pt;
    script[1].comps_in_scan = 1; script[1].component_index[0] = 1;
    script[1].Ss = 8 - psv; script[1].Se = 0; script[1].Ah = 0; script[1].Al = 0;
    c.scan_info = script; c.num_scans = 2;
  } else
    jpeg_enable_lossless(&c, psv, pt);
  jpeg_mem_dest(&c, &out, &outsize);
  jpeg_start_compress(&c, TRUE);
  /* a lossy object's derived state is not what this driver checks: only that lossless mode was turned off */
  if (variant == PROGRESSIVE) printf("  lossless %d\n", c.master->lossless);
  else print_state(&c);
  while (c.next_scanline < c.image_height) {
    JDIMENSION n = c.image_height - c.next_scanline < (JDIMENSION)step ? c.image_height - c.next_scanline : (JDIMENSION)step;
    if (prec == 8) {
      JSAMPROW rows[8];
      for (JDIMENSION r = 0; r < n; r++) rows[r] = pix8 + (size_t)(c.next_scanline + r) * W * nc;
      jpeg_write_scanlines(&c, rows, n);
    } else if (prec == 12) {
      J12SAMPROW rows[8];
      for (JDIMENSION r = 0; r < n; r++) rows[r] = (J12SAMPROW)(pix + (size_t)(c.next_scanline + r) * W * nc);
      jpeg12_write_scanlines(&c, rows, n);
    } else {
      J16SAMPROW rows[8];
      for (JDIMENSION r = 0; r < n; r++) rows[r] = (J16SAMPROW)(pix + (size_t)(c.next_scanline + r) * W * nc);
      jpeg16_write_scanlines(&c, rows, n);
    }
  }
  jpeg_finish_compress(&c);
  printf("  global_state %d bytes %lu hash %016llx\n", c.global_state, outsize, fnv(out, outsize));
  jpeg_destroy_compress(&c);
  free(out); free(pix); free(pix8);
}

static void tj_encode(int prec, int pf, int psv, int pt, int restart_rows)
{
  tjhandle tj = tj3Init(TJINIT_COMPRESS);
  const int nc = tjPixelSize[pf];
  unsigned short *pix = malloc(sizeof(unsigned short) * W * H * nc);
  unsigned char *pix8 = malloc((size_t)W * H * nc);
  unsigned char *out = NULL;
  size_t n = 0;
  int rc;
  fill(pix, W * H, nc, prec, (unsigned)(pf * 17 + psv));
  for (int i = 0; i < W * H * nc; i++) pix8[i] = (unsigned char)pix[i];
  tj3Set(tj, TJPARAM_PRECISION, prec);
  tj3Set(tj, TJPARAM_LOSSLESS, 1);
  tj3Set(tj, TJPARAM_LOSSLESSPSV, psv);
  tj3Set(tj, TJPARAM_LOSSLESSPT, pt);
  tj3Set(tj, TJPARAM_RESTARTROWS, restart_rows);
  if (prec == 8) rc = tj3Compress8(tj, pix8, W, 0, H, pf, &out, &n);
  else if (prec == 12) rc = tj3Compress12(tj, (const short *)pix, W, 0, H, pf, &out, &n);
  else rc = tj3Compress16(tj, pix, W, 0, H, pf, &out, &n);
  if (rc) printf("tj3Compress%d pf %d psv %d pt %d restart %d: error %s\n", prec, pf, psv, pt, restart_rows, tj3GetErrorStr(tj));
  else printf("tj3Compress%d pf %d psv %d pt %d restart %d: bytes %zu hash %016llx\n", prec, pf, psv, pt, restart_rows, n, fnv(out, n));
  tj3Free(out);
  tj3Destroy(tj);
  free(pix); free(pix8);
}

int main(void)
{
  const int pfs[] = {TJPF_RGB, TJPF_BGRX, TJPF_XRGB, TJPF_GRAY};
  const int precs[] = {8, 12, 16};
  for (int k = 0; k < 3; k++)
    for (int f = 0; f < 4; f++)
      tj_encode(precs[k], pfs[f], 1 + (k * 4 + f) % 7, (k + f) % 3, f == 1 ? 2 : 0);
  api_encode("8-bit RGB, psv 4, Pt 1, restart 2 rows", 8, JCS_RGB, 3, 4, 1, 2, PLAIN, 5);
  api_encode("12-bit gray, psv 6", 12, JCS_GRAYSCALE, 1, 6, 0, 0, PLAIN, 3);
  api_encode("16-bit RGB, psv 7, Pt 2, restart 1 row", 16, JCS_RGB, 3, 7, 2, 1, PLAIN, 8);
  api_encode("16-bit CMYK, psv 1", 16, JCS_CMYK, 4, 1, 0, 0, PLAIN, 1);
  api_encode("raw_data_in before jpeg_enable_lossless, 8-bit RGB, psv 2", 8, JCS_RGB, 3, 2, 0, 0, RAW_FIRST, 4);
  api_encode("raw_data_in before jpeg_enable_lossless, 12-bit RGB, psv 3", 12, JCS_RGB, 3, 3, 0, 0, RAW_FIRST, 4);
  api_encode("grayscale, 2x2 sampling, smoothing and no optimize_coding overridden, 8-bit RGB, psv 5", 8, JCS_RGB, 3, 5, 0, 0, OVERRIDES, 6);
  api_encode("hand-made two-scan script, 16-bit RGB, psv 3, Pt 4", 16, JCS_RGB, 3, 3, 4, 0, SCRIPT, 7);
  api_encode("progressive script over jpeg_enable_lossless, 8-bit RGB", 8, JCS_RGB, 3, 1, 0, 0, PROGRESSIVE, 8);
  return 0;
}
