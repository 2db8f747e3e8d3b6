/*
 * tests/refll.c -- TEST INFRASTRUCTURE (not product code).
 *
 * A driver around the unmodified reference library (oracle/_ref/libjpeg_ref.so) for the lossless tests: cjpeg's call
 * order (cjpeg.c main) with -lossless and -precision 16, any input colour space the library accepts (4-component
 * input included, which the cjpeg binary cannot read), 8-, 12- and 16-bit samples, and a hand-made scan script in
 * place of -scans.  __graft_entry__.build() compiles it to build/librefll.so when the reference build is present.
 *
 *   in_color_space = RGB ; jpeg_set_defaults ; switches(for_real = 0)
 *   in_color_space / input_components / size ; jpeg_default_colorspace ; switches(for_real = 1)
 *   (jpeg_simple_progression, jpeg_enable_lossless, the script -- cjpeg.c:747-761) ; start / write / finish
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <setjmp.h>
#include <jpeglib.h>

struct err_mgr { struct jpeg_error_mgr pub; jmp_buf jb; char msg[JMSG_LENGTH_MAX]; };
static void on_error(j_common_ptr c) { struct err_mgr *e = (struct err_mgr *)c->err; (*c->err->format_message)(c, e->msg); longjmp(e->jb, 1); }
static void on_message(j_common_ptr c, int lvl) { (void)c; (void)lvl; }

static int is_opt(const char *a, const char *name) { return a[0] == '-' && !strcmp(a + 1, name); }

/* The subset of cjpeg's switches (cjpeg.c parse_switches) the lossless tests use; returns -1 on an unknown one. */
static int apply_switches(j_compress_ptr c, int argc, const char *const *argv, int for_real, int nscans, const int *script,
                          jpeg_scan_info *scan_buf)
{
  int simple_progressive = c->num_scans != 0, i, ci, psv = 0, pt = 0;
  const char *sample = NULL;
  for (i = 0; i < argc; i++) {
    const char *a = argv[i];
    if (is_opt(a, "baseline")) { simple_progressive = 0; c->num_scans = 0; c->scan_info = NULL; }
    else if (is_opt(a, "revert")) { jpeg_c_set_int_param(c, JINT_COMPRESS_PROFILE, JCP_FASTEST); jpeg_set_defaults(c); }
    else if (is_opt(a, "optimize")) c->optimize_coding = TRUE;
    else if (is_opt(a, "progressive")) simple_progressive = 1;
    else if (is_opt(a, "notrellis")) jpeg_c_set_bool_param(c, JBOOLEAN_TRELLIS_QUANT, FALSE);
    else if (is_opt(a, "grayscale")) jpeg_set_colorspace(c, JCS_GRAYSCALE);
    else if (is_opt(a, "rgb")) jpeg_set_colorspace(c, JCS_RGB);
    else if (is_opt(a, "sample") && i + 1 < argc) sample = argv[++i];
    else if (is_opt(a, "smooth") && i + 1 < argc) c->smoothing_factor = atoi(argv[++i]);
    else if (is_opt(a, "restart") && i + 1 < argc) {                 /* N rows, or NB MCUs */
      const char *v = argv[++i]; const size_t n = strlen(v);
      if (n && (v[n - 1] == 'b' || v[n - 1] == 'B')) { c->restart_interval = (unsigned)atoi(v); c->restart_in_rows = 0; }
      else c->restart_in_rows = atoi(v);
    }
    else if (is_opt(a, "precision") && i + 1 < argc) { c->data_precision = atoi(argv[++i]); }
    else if (is_opt(a, "lossless") && i + 1 < argc) {                /* psv[,Pt] (cjpeg.c:459-480) */
      const char *v = argv[++i], *comma = strchr(v, ',');
      psv = atoi(v); pt = comma ? atoi(comma + 1) : 0;
    } else return -1;
  }
  if (!for_real) return 0;
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
  if (psv != 0) jpeg_enable_lossless(c, psv, pt);
  if (nscans > 0) {                                                   /* read_scan_script (rdswitch.c:244-266) */
    for (i = 0; i < nscans; i++) {
      const int *e = script + 9 * i;
      scan_buf[i].comps_in_scan = e[0];
      for (ci = 0; ci < 4; ci++) scan_buf[i].component_index[ci] = e[1 + ci];
      scan_buf[i].Ss = e[5]; scan_buf[i].Se = e[6]; scan_buf[i].Ah = e[7]; scan_buf[i].Al = e[8];
    }
    c->scan_info = scan_buf; c->num_scans = nscans;
    jpeg_c_set_bool_param(c, JBOOLEAN_OPTIMIZE_SCANS, FALSE);
  }
  return 0;
}

/*
 * Encode one image.  pixels: interleaved samples (uint8 at 8 bits, int16 at 12, uint16 at 16), pitch in samples.
 * script: nscans entries of 9 ints {comps_in_scan, component_index[4], Ss, Se, Ah, Al}.  Returns 0, or -1 with the
 * reference's message in errbuf.
 */
int refll_encode(const void *pixels, int pitch_samples, int width, int height, int in_color_space, int input_components,
                 int argc, const char *const *argv, int nscans, const int *script,
                 unsigned char **out, unsigned long *outsize, char *errbuf, int errlen)
{
  struct jpeg_compress_struct c;
  struct err_mgr e;
  static jpeg_scan_info scan_buf[64];
  *out = NULL; *outsize = 0;
  if (nscans > 64) { snprintf(errbuf, errlen, "too many scans"); return -1; }
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
  if (apply_switches(&c, argc, argv, 0, 0, NULL, scan_buf)) { snprintf(errbuf, errlen, "unknown switch"); jpeg_destroy_compress(&c); return -1; }
  c.in_color_space = (J_COLOR_SPACE)in_color_space; c.input_components = input_components;
  c.image_width = width; c.image_height = height;
  jpeg_default_colorspace(&c);
  apply_switches(&c, argc, argv, 1, nscans, script, scan_buf);
  jpeg_mem_dest(&c, out, outsize);
  jpeg_start_compress(&c, TRUE);
  while (c.next_scanline < c.image_height) {
    if (c.data_precision == 16) {
      J16SAMPROW row = (J16SAMPROW)((const unsigned short *)pixels + (size_t)c.next_scanline * pitch_samples);
      jpeg16_write_scanlines(&c, &row, 1);
    } else if (c.data_precision == 12) {
      J12SAMPROW row = (J12SAMPROW)((const short *)pixels + (size_t)c.next_scanline * pitch_samples);
      jpeg12_write_scanlines(&c, &row, 1);
    } else {
      JSAMPROW row = (JSAMPROW)((const unsigned char *)pixels + (size_t)c.next_scanline * pitch_samples);
      jpeg_write_scanlines(&c, &row, 1);
    }
  }
  jpeg_finish_compress(&c);
  jpeg_destroy_compress(&c);
  return 0;
}

void refll_free(void *p) { free(p); }
