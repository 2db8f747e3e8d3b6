/*
 * tests/refcs.c -- TEST INFRASTRUCTURE (not product code).
 *
 * A small driver around the unmodified reference library (oracle/_ref/libjpeg_ref.so and libturbojpeg_ref.so) for
 * the colour-space tests: encodes of any (in_color_space, jpeg_color_space) pair the reference accepts, from
 * interleaved pixels or from raw-data planes, with cjpeg's call order, and the TurboJPEG entry point tj3Compress8.
 * __graft_entry__.build() compiles it to build/librefcs.so when the reference build is present.
 *
 * The cjpeg sequence (cjpeg.c main) with the colour spaces of the image header made explicit:
 *   in_color_space = RGB ; jpeg_set_defaults ; switches(for_real = 0)
 *   in_color_space / input_components / size from the "header" ; jpeg_default_colorspace
 *   jpeg_set_colorspace(jpeg_color_space) when one is given ; switches(for_real = 1) ; start / write / finish
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <setjmp.h>
#include <jpeglib.h>
#include <turbojpeg.h>

struct err_mgr { struct jpeg_error_mgr pub; jmp_buf jb; char msg[JMSG_LENGTH_MAX]; };
static void on_error(j_common_ptr c) { struct err_mgr *e = (struct err_mgr *)c->err; (*c->err->format_message)(c, e->msg); longjmp(e->jb, 1); }
static void on_message(j_common_ptr c, int lvl) { (void)c; (void)lvl; }

static int is_opt(const char *a, const char *name) { return a[0] == '-' && !strcmp(a + 1, name); }

/* The subset of cjpeg's switches (cjpeg.c parse_switches) the colour-space tests use; returns -1 on an unknown one. */
static int apply_switches(j_compress_ptr c, int argc, const char *const *argv, int for_real)
{
  int force_baseline = 0, simple_progressive = c->num_scans != 0, i, ci;
  double quality = -1.0;
  const char *sample = NULL;
  for (i = 0; i < argc; i++) {
    const char *a = argv[i];
    if (is_opt(a, "baseline")) { force_baseline = 1; simple_progressive = 0; c->num_scans = 0; c->scan_info = NULL; }
    else if (is_opt(a, "revert")) { jpeg_c_set_int_param(c, JINT_COMPRESS_PROFILE, JCP_FASTEST); jpeg_set_defaults(c); }
    else if (is_opt(a, "optimize")) c->optimize_coding = TRUE;
    else if (is_opt(a, "progressive")) simple_progressive = 1;
    else if (is_opt(a, "fastcrush")) jpeg_c_set_bool_param(c, JBOOLEAN_OPTIMIZE_SCANS, FALSE);
    else if (is_opt(a, "notrellis")) jpeg_c_set_bool_param(c, JBOOLEAN_TRELLIS_QUANT, FALSE);
    else if (is_opt(a, "noovershoot")) jpeg_c_set_bool_param(c, JBOOLEAN_OVERSHOOT_DERINGING, FALSE);
    else if (is_opt(a, "quality") && i + 1 < argc) quality = atof(argv[++i]);
    else if (is_opt(a, "sample") && i + 1 < argc) sample = argv[++i];
    else if (is_opt(a, "smooth") && i + 1 < argc) c->smoothing_factor = atoi(argv[++i]);
    else if (is_opt(a, "restart") && i + 1 < argc) {                 /* N rows, or NB MCUs */
      const char *v = argv[++i]; const size_t n = strlen(v);
      if (n && (v[n - 1] == 'b' || v[n - 1] == 'B')) { c->restart_interval = (unsigned)atoi(v); c->restart_in_rows = 0; }
      else c->restart_in_rows = atoi(v);
    }
    else if (is_opt(a, "precision") && i + 1 < argc) { if (!for_real) c->data_precision = atoi(argv[i + 1]); i++; }
    else if (is_opt(a, "dct") && i + 1 < argc) {
      const char *m = argv[++i];
      c->dct_method = !strcmp(m, "fast") ? JDCT_IFAST : !strcmp(m, "float") ? JDCT_FLOAT : JDCT_ISLOW;
    } else return -1;
  }
  if (!for_real) return 0;
  if (quality >= 0) {
    /* set_quality_ratings with one value: both table slots scaled alike, then the mozjpeg sampling defaults */
    jpeg_set_linear_quality(c, (int)jpeg_float_quality_scaling((float)quality), force_baseline);
    if (quality >= 90) { for (ci = 0; ci < MAX_COMPONENTS; ci++) c->comp_info[ci].h_samp_factor = c->comp_info[ci].v_samp_factor = 1; }
    else if (quality >= 80) {
      c->comp_info[0].h_samp_factor = 2; c->comp_info[0].v_samp_factor = 1;
      for (ci = 1; ci < MAX_COMPONENTS; ci++) c->comp_info[ci].h_samp_factor = c->comp_info[ci].v_samp_factor = 1;
    }
  }
  if (sample) {
    /* set_sample_factors: the listed components, 1x1 for the rest */
    const char *s = sample;
    for (ci = 0; ci < MAX_COMPONENTS; ci++) {
      int h = 1, v = 1;
      if (*s) { if (sscanf(s, "%dx%d", &h, &v) != 2) return -1; while (*s && *s != ',') s++; if (*s == ',') s++; }
      c->comp_info[ci].h_samp_factor = h; c->comp_info[ci].v_samp_factor = v;
    }
  }
  if (simple_progressive) jpeg_simple_progression(c);
  return 0;
}

/*
 * Encode one image.  pixels: interleaved samples (uint8, or uint16 at 12 bits), pitch in samples; or, with
 * planes != NULL, jpeg_write_raw_data input: planes[ci] holds height_in_blocks*8 rows of pitch[ci] samples.
 * jpeg_color_space < 0: the default for in_color_space.  Returns 0, or -1 with the reference's message in errbuf.
 */
int refcs_encode(const void *pixels, int pitch_samples, const unsigned char *const *planes, const int *pitch,
                 int width, int height, int in_color_space, int input_components, int jpeg_color_space,
                 int argc, const char *const *argv, unsigned char **out, unsigned long *outsize, char *errbuf, int errlen)
{
  struct jpeg_compress_struct c;
  struct err_mgr e;
  *out = NULL; *outsize = 0;
  c.err = jpeg_std_error(&e.pub);
  e.pub.error_exit = on_error; e.pub.emit_message = on_message;
  if (setjmp(e.jb)) {
    snprintf(errbuf, errlen, "%s", e.msg);
    jpeg_destroy_compress(&c);
    if (*out) { free(*out); *out = NULL; }
    return -1;
  }
  jpeg_create_compress(&c);
  c.in_color_space = JCS_RGB; c.input_components = 3;
  jpeg_set_defaults(&c);
  if (apply_switches(&c, argc, argv, 0)) { snprintf(errbuf, errlen, "unknown switch"); jpeg_destroy_compress(&c); return -1; }
  c.in_color_space = (J_COLOR_SPACE)in_color_space; c.input_components = input_components;
  c.image_width = width; c.image_height = height;
  jpeg_default_colorspace(&c);
  if (jpeg_color_space >= 0) jpeg_set_colorspace(&c, (J_COLOR_SPACE)jpeg_color_space);
  apply_switches(&c, argc, argv, 1);
  c.raw_data_in = planes != NULL;
  jpeg_mem_dest(&c, out, outsize);
  jpeg_start_compress(&c, TRUE);
  if (planes) {
    JSAMPROW rows[MAX_COMPONENTS][4 * DCTSIZE]; JSAMPARRAY data[MAX_COMPONENTS];
    const int lines = c.max_v_samp_factor * DCTSIZE;
    int ci, r;
    for (ci = 0; ci < c.num_components; ci++) data[ci] = rows[ci];
    while (c.next_scanline < c.image_height) {
      const int imcu = c.next_scanline / lines;
      for (ci = 0; ci < c.num_components; ci++) {
        const int v = c.comp_info[ci].v_samp_factor, last = (int)c.comp_info[ci].height_in_blocks * DCTSIZE - 1;
        for (r = 0; r < v * DCTSIZE; r++) { int y = imcu * v * DCTSIZE + r; rows[ci][r] = (JSAMPROW)(planes[ci] + (size_t)(y < last ? y : last) * pitch[ci]); }
      }
      jpeg_write_raw_data(&c, data, lines);
    }
  } else if (c.data_precision == 12) {
    while (c.next_scanline < c.image_height) {
      J12SAMPROW row = (J12SAMPROW)((const short *)pixels + (size_t)c.next_scanline * pitch_samples);
      jpeg12_write_scanlines(&c, &row, 1);
    }
  } else {
    while (c.next_scanline < c.image_height) {
      JSAMPROW row = (JSAMPROW)((const unsigned char *)pixels + (size_t)c.next_scanline * pitch_samples);
      jpeg_write_scanlines(&c, &row, 1);
    }
  }
  jpeg_finish_compress(&c);
  jpeg_destroy_compress(&c);
  return 0;
}

/* tj3Compress8 on TJPF_CMYK pixels (4 samples per pixel, rows packed).  colorspace: a TJCS_* value, or -1 for the
 * library's choice (YCCK).  subsamp: a TJSAMP_* value. */
int refcs_encode_tj_cmyk(const unsigned char *pixels, int width, int height, int quality, int subsamp, int optimize,
                         int progressive, int colorspace, unsigned char **out, unsigned long *outsize, char *errbuf, int errlen)
{
  tjhandle h = tj3Init(TJINIT_COMPRESS);
  size_t size = 0;
  int rc = -1;
  *out = NULL; *outsize = 0;
  if (!h) { snprintf(errbuf, errlen, "tj3Init failed"); return -1; }
  if (tj3Set(h, TJPARAM_QUALITY, quality) || tj3Set(h, TJPARAM_SUBSAMP, subsamp) || tj3Set(h, TJPARAM_OPTIMIZE, optimize) ||
      tj3Set(h, TJPARAM_PROGRESSIVE, progressive) || (colorspace >= 0 && tj3Set(h, TJPARAM_COLORSPACE, colorspace)))
    snprintf(errbuf, errlen, "%s", tj3GetErrorStr(h));
  else if (tj3Compress8(h, pixels, width, 0, height, TJPF_CMYK, out, &size))
    snprintf(errbuf, errlen, "%s", tj3GetErrorStr(h));
  else { *outsize = (unsigned long)size; rc = 0; }
  tj3Destroy(h);
  return rc;
}

void refcs_free(void *p) { free(p); }
void refcs_tjfree(void *p) { tj3Free(p); }
