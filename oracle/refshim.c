/*
 * oracle/refshim.c -- TEST INFRASTRUCTURE (not product code).
 *
 * A thin driver around the UNMODIFIED reference library (oracle/_ref/
 * libjpeg_ref.so, compiled from /root/reference by oracle/Makefile).  It lets
 * the tests and bench.py's cpu_baseline leg run the reference encoder on an
 * in-memory RGB buffer with the same switch semantics as the reference's cjpeg
 * front end (cjpeg.c:315-765), without going through PPM files.
 *
 * The order of API calls below mirrors what `cjpeg` does for the equivalent
 * command line (cjpeg.c main(): create -> in_color_space -> set_defaults ->
 * parse_switches(dummy) -> image dims -> default_colorspace ->
 * parse_switches(for_real) -> start/write/finish).
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <setjmp.h>
#include <jpeglib.h>

typedef struct {
  int revert;          /* -revert                     */
  int baseline;        /* -baseline                   */
  int has_quality;     /* -quality given              */
  float quality;       /* -quality N                  */
  int samp_h[4], samp_v[4]; /* -sample HxV,... ; samp_h[0]==0 => not given */
  int optimize;        /* -optimize                   */
  int progressive;     /* -progressive                */
  int fastcrush;       /* -fastcrush                  */
  int notrellis;       /* -notrellis                  */
  int trellis_dc;      /* 1: -trellis-dc, 0: -notrellis-dc, -1: leave default */
  int noovershoot;     /* -noovershoot                */
  int dct;             /* 0 int, 1 fast, 2 float, -1 default */
  int restart;         /* -restart N  (rows) or N with restart_blocks */
  int restart_blocks;  /* 1 => value is in MCUs ('B' suffix) */
  int grayscale;       /* -grayscale                  */
  int quant_table;     /* -quant-table N, -1 not given */
  int precision;       /* 8 or 12                     */
  int has_lambda1, has_lambda2;
  float lambda1, lambda2;
  int tjapi;           /* 1: emulate TurboJPEG tj3Compress8 parameter setup
                          (turbojpeg.c:330-397): JCP_FASTEST, quality,
                          subsampling from samp_h/v[0], optimize/progressive */
  int input_gray;      /* input buffer is 1 component grayscale */
  /* extension parameters cjpeg has no switch for (jpeg_c_set_*_param, jcext.c); -1 = leave the default */
  int ext_use_scans_in_trellis, ext_trellis_freq_split, ext_trellis_eob_opt, ext_trellis_q_opt, ext_trellis_num_loops;
  int has_dc_ver_weight; float dc_ver_weight;   /* -trellis-dc-ver-weight W (cjpeg.c:667-672) */
} refshim_cfg;

struct my_err { struct jpeg_error_mgr pub; jmp_buf jb; char msg[JMSG_LENGTH_MAX]; };
static void my_exit(j_common_ptr c) {
  struct my_err *e = (struct my_err *)c->err;
  (*c->err->format_message)(c, e->msg);
  longjmp(e->jb, 1);
}
static void my_emit(j_common_ptr c, int lvl) { (void)c; (void)lvl; }

static void apply_switches(j_compress_ptr cinfo, const refshim_cfg *cfg, int for_real,
                           int *force_baseline, int *simple_progressive)
{
  *force_baseline = 0;
  *simple_progressive = cinfo->num_scans == 0 ? 0 : 1;   /* cjpeg.c:343 */
  if (cfg->revert) {                                     /* cjpeg.c:623-626 */
    jpeg_c_set_int_param(cinfo, JINT_COMPRESS_PROFILE, JCP_FASTEST);
    jpeg_set_defaults(cinfo);
  }
  if (cfg->baseline) {                                   /* cjpeg.c:378-384 */
    *force_baseline = 1; *simple_progressive = 0;
    cinfo->num_scans = 0; cinfo->scan_info = NULL;
  }
  if (cfg->dct == 0) cinfo->dct_method = JDCT_ISLOW;
  else if (cfg->dct == 1) cinfo->dct_method = JDCT_IFAST;
  else if (cfg->dct == 2) cinfo->dct_method = JDCT_FLOAT;
  if (cfg->fastcrush) jpeg_c_set_bool_param(cinfo, JBOOLEAN_OPTIMIZE_SCANS, FALSE);
  if (cfg->grayscale) jpeg_set_colorspace(cinfo, JCS_GRAYSCALE);
  if (cfg->ext_use_scans_in_trellis >= 0) jpeg_c_set_bool_param(cinfo, JBOOLEAN_USE_SCANS_IN_TRELLIS, cfg->ext_use_scans_in_trellis);
  if (cfg->ext_trellis_freq_split >= 0) jpeg_c_set_int_param(cinfo, JINT_TRELLIS_FREQ_SPLIT, cfg->ext_trellis_freq_split);
  if (cfg->ext_trellis_eob_opt >= 0) jpeg_c_set_bool_param(cinfo, JBOOLEAN_TRELLIS_EOB_OPT, cfg->ext_trellis_eob_opt);
  if (cfg->ext_trellis_q_opt >= 0) jpeg_c_set_bool_param(cinfo, JBOOLEAN_TRELLIS_Q_OPT, cfg->ext_trellis_q_opt);
  if (cfg->ext_trellis_num_loops >= 0) jpeg_c_set_int_param(cinfo, JINT_TRELLIS_NUM_LOOPS, cfg->ext_trellis_num_loops);
  if (cfg->has_dc_ver_weight) jpeg_c_set_float_param(cinfo, JFLOAT_TRELLIS_DELTA_DC_WEIGHT, cfg->dc_ver_weight);
  if (cfg->has_lambda1) jpeg_c_set_float_param(cinfo, JFLOAT_LAMBDA_LOG_SCALE1, cfg->lambda1);
  if (cfg->has_lambda2) jpeg_c_set_float_param(cinfo, JFLOAT_LAMBDA_LOG_SCALE2, cfg->lambda2);
  if (cfg->optimize) cinfo->optimize_coding = TRUE;
  if (cfg->progressive) *simple_progressive = 1;
  if (cfg->quant_table >= 0) {                           /* cjpeg.c:585-596 */
    jpeg_c_set_int_param(cinfo, JINT_BASE_QUANT_TBL_IDX, cfg->quant_table);
    jpeg_set_quality(cinfo, 75, TRUE);
  }
  if (cfg->restart > 0) {
    if (cfg->restart_blocks) { cinfo->restart_interval = cfg->restart; cinfo->restart_in_rows = 0; }
    else cinfo->restart_in_rows = cfg->restart;
  }
  if (cfg->trellis_dc == 0) jpeg_c_set_bool_param(cinfo, JBOOLEAN_TRELLIS_QUANT_DC, FALSE);
  if (cfg->notrellis) jpeg_c_set_bool_param(cinfo, JBOOLEAN_TRELLIS_QUANT, FALSE);
  if (cfg->trellis_dc == 1) jpeg_c_set_bool_param(cinfo, JBOOLEAN_TRELLIS_QUANT_DC, TRUE);
  if (cfg->noovershoot) jpeg_c_set_bool_param(cinfo, JBOOLEAN_OVERSHOOT_DERINGING, FALSE);

  if (for_real) {
    int ci;
    if (cfg->has_quality) {
      /* rdswitch.c:524-573 set_quality_ratings with a single value */
      int sf = (int)jpeg_float_quality_scaling(cfg->quality);
      int idx = jpeg_c_get_int_param(cinfo, JINT_BASE_QUANT_TBL_IDX);
      (void)idx;
      /* jpeg_default_qtables (rdswitch.c:509-521) == jpeg_set_linear_quality
         with the master table index; both slots get the same factor here. */
      jpeg_set_linear_quality(cinfo, sf, *force_baseline);
      if (cfg->quality >= 90) {
        for (ci = 0; ci < MAX_COMPONENTS; ci++) { cinfo->comp_info[ci].h_samp_factor = 1; cinfo->comp_info[ci].v_samp_factor = 1; }
      } else if (cfg->quality >= 80) {
        cinfo->comp_info[0].h_samp_factor = 2; cinfo->comp_info[0].v_samp_factor = 1;
        for (ci = 1; ci < MAX_COMPONENTS; ci++) { cinfo->comp_info[ci].h_samp_factor = 1; cinfo->comp_info[ci].v_samp_factor = 1; }
      }
    }
    if (cfg->samp_h[0] > 0) {
      /* rdswitch.c set_sample_factors: listed comps, rest default to 1x1 */
      for (ci = 0; ci < MAX_COMPONENTS; ci++) {
        int h = 1, v = 1;
        if (ci < 4 && cfg->samp_h[ci] > 0) { h = cfg->samp_h[ci]; v = cfg->samp_v[ci]; }
        cinfo->comp_info[ci].h_samp_factor = h; cinfo->comp_info[ci].v_samp_factor = v;
      }
    }
    if (*simple_progressive) jpeg_simple_progression(cinfo);
  }
}

/* Returns 0 on success; *out is malloc'ed (free with refshim_free). */
int refshim_encode(const void *pixels, int width, int height, int pitch_samples,
                   const refshim_cfg *cfg, unsigned char **out, unsigned long *outsize,
                   char *errbuf, int errbuf_len)
{
  struct jpeg_compress_struct cinfo;
  struct my_err jerr;
  int fb, sp;
  *out = NULL; *outsize = 0;
  cinfo.err = jpeg_std_error(&jerr.pub);
  jerr.pub.error_exit = my_exit;
  jerr.pub.emit_message = my_emit;
  if (setjmp(jerr.jb)) {
    if (errbuf && errbuf_len > 0) { strncpy(errbuf, jerr.msg, errbuf_len - 1); errbuf[errbuf_len - 1] = 0; }
    jpeg_destroy_compress(&cinfo);
    if (*out) { free(*out); *out = NULL; }
    return -1;
  }
  jpeg_create_compress(&cinfo);
  if (cfg->tjapi) {
    /* turbojpeg.c:330-397 setCompDefaults */
    int ci;
    cinfo.in_color_space = cfg->input_gray ? JCS_GRAYSCALE : JCS_RGB;
    cinfo.input_components = cfg->input_gray ? 1 : 3;
    jpeg_c_set_int_param(&cinfo, JINT_COMPRESS_PROFILE, JCP_FASTEST);
    jpeg_set_defaults(&cinfo);
    cinfo.optimize_coding = cfg->optimize ? TRUE : FALSE;
    cinfo.image_width = width; cinfo.image_height = height;
    jpeg_set_quality(&cinfo, (int)cfg->quality, TRUE);
    cinfo.dct_method = (cfg->dct == 1) ? JDCT_FASTEST : JDCT_ISLOW;
    jpeg_set_colorspace(&cinfo, (cfg->grayscale || cfg->input_gray) ? JCS_GRAYSCALE : JCS_YCbCr);
    if (cfg->progressive) jpeg_simple_progression(&cinfo);
    cinfo.comp_info[0].h_samp_factor = cfg->samp_h[0] > 0 ? cfg->samp_h[0] : 1;
    cinfo.comp_info[0].v_samp_factor = cfg->samp_h[0] > 0 ? cfg->samp_v[0] : 1;
    for (ci = 1; ci < cinfo.num_components; ci++) { cinfo.comp_info[ci].h_samp_factor = 1; cinfo.comp_info[ci].v_samp_factor = 1; }
    if (cfg->restart > 0) { if (cfg->restart_blocks) cinfo.restart_interval = cfg->restart; else cinfo.restart_in_rows = cfg->restart; }
  } else {
    cinfo.in_color_space = cfg->input_gray ? JCS_GRAYSCALE : JCS_RGB;   /* cjpeg.c:860 */
    cinfo.input_components = cfg->input_gray ? 1 : 3;
    jpeg_set_defaults(&cinfo);
    apply_switches(&cinfo, cfg, 0, &fb, &sp);
    if (cfg->precision == 12) cinfo.data_precision = 12;
    cinfo.image_width = width; cinfo.image_height = height;
    jpeg_default_colorspace(&cinfo);                                      /* cjpeg.c:931 */
    apply_switches(&cinfo, cfg, 1, &fb, &sp);
  }
  jpeg_mem_dest(&cinfo, out, outsize);
  jpeg_start_compress(&cinfo, TRUE);
  if (cinfo.data_precision == 12) {
    const short *p = (const short *)pixels;
    while (cinfo.next_scanline < cinfo.image_height) {
      J12SAMPROW row = (J12SAMPROW)(p + (size_t)cinfo.next_scanline * pitch_samples);
      jpeg12_write_scanlines(&cinfo, &row, 1);
    }
  } else {
    const unsigned char *p = (const unsigned char *)pixels;
    while (cinfo.next_scanline < cinfo.image_height) {
      JSAMPROW row = (JSAMPROW)(p + (size_t)cinfo.next_scanline * pitch_samples);
      jpeg_write_scanlines(&cinfo, &row, 1);
    }
  }
  jpeg_finish_compress(&cinfo);
  jpeg_destroy_compress(&cinfo);
  return 0;
}

/* The same through jpeg_write_raw_data: planes[ci] = hib*8 rows of wib*8 samples (pitch in samples). */
int refshim_encode_raw(const unsigned char *const *planes, const int *pitch, int width, int height, int ncomp,
                       const refshim_cfg *cfg, unsigned char **out, unsigned long *outsize, char *errbuf, int errlen)
{
  struct jpeg_compress_struct cinfo;
  struct my_err jerr;
  int fb = 0, sp = 0, ci;
  *out = NULL; *outsize = 0;
  cinfo.err = jpeg_std_error(&jerr.pub);
  jerr.pub.error_exit = my_exit;
  if (setjmp(jerr.jb)) { (*cinfo.err->format_message)((j_common_ptr)&cinfo, jerr.msg); snprintf(errbuf, errlen, "%s", jerr.msg); jpeg_destroy_compress(&cinfo); return 1; }
  jpeg_create_compress(&cinfo);
  cinfo.in_color_space = ncomp == 1 ? JCS_GRAYSCALE : JCS_YCbCr;      /* raw data: the planes are already in the JPEG colour space */
  cinfo.input_components = ncomp;
  jpeg_set_defaults(&cinfo);
  apply_switches(&cinfo, cfg, 0, &fb, &sp);
  cinfo.image_width = width; cinfo.image_height = height;
  jpeg_default_colorspace(&cinfo);
  apply_switches(&cinfo, cfg, 1, &fb, &sp);
  cinfo.raw_data_in = TRUE;
  jpeg_mem_dest(&cinfo, out, outsize);
  jpeg_start_compress(&cinfo, TRUE);
  {
    JSAMPROW rows[3][32]; JSAMPARRAY data[3];
    int lines = cinfo.max_v_samp_factor * DCTSIZE;
    for (ci = 0; ci < ncomp; ci++) data[ci] = rows[ci];
    while (cinfo.next_scanline < cinfo.image_height) {
      int imcu = cinfo.next_scanline / lines, r;
      for (ci = 0; ci < ncomp; ci++) {
        int v = cinfo.comp_info[ci].v_samp_factor, hrows = (int)cinfo.comp_info[ci].height_in_blocks * DCTSIZE;
        for (r = 0; r < v * DCTSIZE; r++) { int y = imcu * v * DCTSIZE + r; if (y > hrows - 1) y = hrows - 1; rows[ci][r] = (JSAMPROW)(planes[ci] + (size_t)y * pitch[ci]); }
      }
      jpeg_write_raw_data(&cinfo, data, lines);
    }
  }
  jpeg_finish_compress(&cinfo);
  jpeg_destroy_compress(&cinfo);
  return 0;
}

void refshim_free(void *p) { free(p); }

/*
 * Decode the quantized coefficient planes of a JPEG (jpeg_read_coefficients).
 * Query mode (coefs == NULL): fills ncomp, wib[], hib[] (blocks), qt[ci][64].
 * coefs[ci] must then hold wib*hib*64 int16 each (natural order per block).
 */
int refshim_read_coefs(const unsigned char *jpg, unsigned long size, int *ncomp,
                       int *wib, int *hib, unsigned short *qt, short **coefs)
{
  struct jpeg_decompress_struct d;
  struct my_err jerr;
  jvirt_barray_ptr *arrs;
  int ci;
  d.err = jpeg_std_error(&jerr.pub);
  jerr.pub.error_exit = my_exit;
  jerr.pub.emit_message = my_emit;
  if (setjmp(jerr.jb)) { jpeg_destroy_decompress(&d); return -1; }
  jpeg_create_decompress(&d);
  jpeg_mem_src(&d, jpg, size);
  jpeg_read_header(&d, TRUE);
  arrs = jpeg_read_coefficients(&d);
  *ncomp = d.num_components;
  for (ci = 0; ci < d.num_components; ci++) {
    jpeg_component_info *c = &d.comp_info[ci];
    int r, i;
    wib[ci] = c->width_in_blocks; hib[ci] = c->height_in_blocks;
    if (qt && c->quant_table) for (i = 0; i < 64; i++) qt[ci * 64 + i] = c->quant_table->quantval[i];
    if (coefs && coefs[ci]) {
      for (r = 0; r < (int)c->height_in_blocks; r++) {
        JBLOCKARRAY b = (*d.mem->access_virt_barray)((j_common_ptr)&d, arrs[ci], r, 1, FALSE);
        memcpy(coefs[ci] + (size_t)r * c->width_in_blocks * 64, b[0], (size_t)c->width_in_blocks * 64 * sizeof(short));
      }
    }
  }
  jpeg_finish_decompress(&d);
  jpeg_destroy_decompress(&d);
  return 0;
}

/*
 * refshim_read_coefs with the number of warnings the reference emitted on the way (corrupt data it decoded anyway:
 * premature end of a segment, an invalid Huffman code, extraneous bytes before a marker, ...) in *warnings.  Returns
 * -1 where the reference stops with an error; *warnings then counts the warnings before it.
 */
static int warn_count;
static void count_emit(j_common_ptr c, int lvl) { (void)c; if (lvl < 0) warn_count++; }

int refshim_read_coefs_warn(const unsigned char *jpg, unsigned long size, int *ncomp,
                            int *wib, int *hib, unsigned short *qt, short **coefs, int *warnings)
{
  struct jpeg_decompress_struct d;
  struct my_err jerr;
  jvirt_barray_ptr *arrs;
  int ci;
  warn_count = 0;
  d.err = jpeg_std_error(&jerr.pub);
  jerr.pub.error_exit = my_exit;
  jerr.pub.emit_message = count_emit;
  if (setjmp(jerr.jb)) { jpeg_destroy_decompress(&d); *warnings = warn_count; return -1; }
  jpeg_create_decompress(&d);
  jpeg_mem_src(&d, jpg, size);
  jpeg_read_header(&d, TRUE);
  arrs = jpeg_read_coefficients(&d);
  *ncomp = d.num_components;
  for (ci = 0; ci < d.num_components; ci++) {
    jpeg_component_info *c = &d.comp_info[ci];
    int r, i;
    wib[ci] = c->width_in_blocks; hib[ci] = c->height_in_blocks;
    if (qt && c->quant_table) for (i = 0; i < 64; i++) qt[ci * 64 + i] = c->quant_table->quantval[i];
    if (coefs && coefs[ci]) {
      for (r = 0; r < (int)c->height_in_blocks; r++) {
        JBLOCKARRAY b = (*d.mem->access_virt_barray)((j_common_ptr)&d, arrs[ci], r, 1, FALSE);
        memcpy(coefs[ci] + (size_t)r * c->width_in_blocks * 64, b[0], (size_t)c->width_in_blocks * 64 * sizeof(short));
      }
    }
  }
  jpeg_finish_decompress(&d);
  jpeg_destroy_decompress(&d);
  *warnings = warn_count;
  return 0;
}

/* Direct access to reference internals used as per-stage oracles. */
extern void jpeg_fdct_islow(int *data);
void refshim_fdct_islow(int *data) { jpeg_fdct_islow(data); }
