/*
 * b200_libjpeg_shim.c -- the reference-side binding of libb200jpeg, as an
 * interposition library for the libjpeg API (JPEG_LIB_VERSION 62).
 *
 * Loaded in front of the reference's libjpeg (LD_PRELOAD, or linked before it),
 * it takes over the calls that bracket the encode hot path,
 *
 *     jpeg_start_compress      (jcapistd.c:44-70)
 *     jpeg_write_scanlines     (jcapistd.c:90-135; jpeg12_write_scanlines for 12-bit samples; 16-bit samples reach the
 *                               device through the reference's own jpeg16_write_scanlines, see device_process_data_16)
 *     jpeg_write_raw_data      (jcapistd.c:145-195; under tj3CompressFromYUV*)
 *     jpeg_write_coefficients  (jctrans.c:39-66; the encode half of jpegtran)
 *     jpeg_finish_compress     (jcapimin.c:176-229)
 *     jpeg_write_marker        (jcapimin.c:232-261; segments are spliced in after the file header)
 *     tj3EncodeYUVPlanes8 / tj3EncodeYUV8  (turbojpeg.c:1467-1690; TurboJPEG's YUV encoding, interposer form only)
 *
 * and runs the image through the C-ABI of include/b200jpeg.h (sm_90a kernels).
 * Everything else -- jpeg_create_compress, jpeg_set_defaults, jpeg_set_quality,
 * jpeg_c_set_*_param, destination managers, error handling -- stays the
 * reference's own code, so an unmodified application (the reference's `cjpeg`
 * binary, in tests/test_libjpeg_shim.py) produces its files on the GPU.
 *
 * Parameter sets the device path does not cover (B200JPEG_ERR_UNSUPPORTED from
 * b200jpeg_start_compress: arithmetic coding, the optional trellis modes, abbreviated
 * datastreams, ...) and hosts without a CUDA device fall through to the reference's
 * implementation of the same three functions (dlsym RTLD_NEXT): that is the
 * REFERENCE running, not a CPU path of this library.  B200_SHIM_VERBOSE=1
 * reports on stderr which path an image took; B200_SHIM_REQUIRE=1 turns a
 * fall-through into error_exit (used by the tests, which must not pass on the
 * reference's code).
 *
 * Built against the reference's own headers (jpeglib.h / jpegint.h and the
 * generated jconfig.h under oracle/_ref/cfg) by integration/Makefile; nothing
 * of the reference is copied into this repository.
 */
#define _GNU_SOURCE
#include <dlfcn.h>
#include <limits.h>
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define JPEG_INTERNALS
#include "jinclude.h"
#include "jpeglib.h"        /* with JPEG_INTERNALS this pulls in jpegint.h and jerror.h */

#include "b200jpeg.h"

#define MAX_ACTIVE 16
static struct {
  j_compress_ptr cinfo; b200jpeg_encoder *enc;
  jvirt_barray_ptr *coef_arrays; b200jpeg_params params;     /* jpeg_write_coefficients objects: read at finish time */
  int raw; uint8_t *plane[4]; size_t plane_pitch[4], plane_rows[4];   /* jpeg_write_raw_data objects: the component planes so far */
  unsigned char *extra; size_t extra_len, extra_cap;         /* jpeg_write_marker segments, in call order */
  size_t header_len;                                         /* SOI + JFIF APP0 + Adobe APP14 (write_file_header, jcmarker.c:649-663) */
  int total_passes;                                          /* what jinit_c_master_control would have counted (jcmaster.c:1114-1139) */
  int lossless;                                              /* a lossless (SOF3) object */
} g_active[MAX_ACTIVE];
static b200jpeg_encoder *g_idle_enc;          /* encoders are reused: creating one costs a CUDA context */
static int g_no_device;
/* libjpeg lets different threads work on different objects (libjpeg.txt, "Multiple-thread usage"): the slot table and
 * the spare encoder are shared, so every access to them is under this lock; a slot's contents belong to the thread
 * that owns the object. */
static pthread_mutex_t g_lock = PTHREAD_MUTEX_INITIALIZER;

static int verbose(void) { const char *v = getenv("B200_SHIM_VERBOSE"); return v && v[0] == '1'; }
static int required(void) { const char *v = getenv("B200_SHIM_REQUIRE"); return v && v[0] == '1'; }

typedef void (*start_fn)(j_compress_ptr, boolean);
typedef JDIMENSION (*write_fn)(j_compress_ptr, JSAMPARRAY, JDIMENSION);
typedef void (*finish_fn)(j_compress_ptr);
typedef void (*abort_fn)(j_compress_ptr);
typedef void (*marker_fn)(j_compress_ptr, int, const JOCTET *, unsigned int);

#ifdef B200_SHIM_STANDALONE
/* Standalone libjpeg.so.62 (integration/Makefile): the reference's unmodified objects are linked into the same library
 * with the entry points this file takes over renamed b200ref_<name> (objcopy --redefine-sym), so "the reference's
 * implementation" is a direct symbol instead of the next library in the search order. */
#define B200REF(n) extern void b200ref_##n(void);
B200REF(jpeg_start_compress) B200REF(jpeg_write_scanlines) B200REF(jpeg12_write_scanlines) B200REF(jpeg_write_raw_data)
B200REF(jpeg_write_coefficients) B200REF(jpeg_finish_compress) B200REF(jpeg_abort_compress) B200REF(jpeg_destroy_compress)
B200REF(jpeg_abort) B200REF(jpeg_destroy) B200REF(jpeg_write_marker) B200REF(jpeg_write_m_header) B200REF(jpeg_write_m_byte)
#undef B200REF
static void *next_sym(const char *name)
{
#define B200REF(n) if (!strcmp(name, #n)) return (void *)b200ref_##n;
  B200REF(jpeg_start_compress) B200REF(jpeg_write_scanlines) B200REF(jpeg12_write_scanlines) B200REF(jpeg_write_raw_data)
  B200REF(jpeg_write_coefficients) B200REF(jpeg_finish_compress) B200REF(jpeg_abort_compress) B200REF(jpeg_destroy_compress)
  B200REF(jpeg_abort) B200REF(jpeg_destroy) B200REF(jpeg_write_marker) B200REF(jpeg_write_m_header) B200REF(jpeg_write_m_byte)
#undef B200REF
  fprintf(stderr, "b200 libjpeg: no reference implementation of %s in this library\n", name); abort();
}
#else
static void *next_sym(const char *name)
{
  void *p = dlsym(RTLD_NEXT, name);
  if (!p) { fprintf(stderr, "b200 shim: the reference's %s is not behind this library\n", name); abort(); }
  return p;
}
#endif

static int find_active(j_compress_ptr cinfo)
{
  int r = -1;
  pthread_mutex_lock(&g_lock);
  for (int i = 0; i < MAX_ACTIVE; i++) if (g_active[i].cinfo == cinfo) { r = i; break; }
  pthread_mutex_unlock(&g_lock);
  return r;
}
/* reusable: the encoder is between images (a finished one); anything else (errors, abandoned objects) destroys it,
 * because its streaming state cannot be reset from outside */
static void release_slot_ex(int i, int reusable)
{
  b200jpeg_encoder *enc = g_active[i].enc, *kill = NULL;
  free(g_active[i].extra);
  for (int k = 0; k < 4; k++) free(g_active[i].plane[k]);
  pthread_mutex_lock(&g_lock);
  if (reusable && !g_idle_enc) g_idle_enc = enc; else kill = enc;
  memset(&g_active[i], 0, sizeof g_active[i]);
  pthread_mutex_unlock(&g_lock);
  if (kill) b200jpeg_encoder_destroy(kill);
}
static void release_slot(int i) { release_slot_ex(i, 0); }
/* a free slot and an encoder for `cinfo` (a stale slot of the same object is dropped first); -1 and *why set when
 * there is none */
static int claim_slot(j_compress_ptr cinfo, const char **why)
{
  int stale = find_active(cinfo);
  if (stale >= 0) release_slot(stale);
  int slot = -1;
  b200jpeg_encoder *enc = NULL;
  pthread_mutex_lock(&g_lock);
  for (int i = 0; i < MAX_ACTIVE && slot < 0; i++) if (!g_active[i].cinfo) slot = i;
  if (slot >= 0) {
    enc = g_idle_enc; g_idle_enc = NULL;
    memset(&g_active[slot], 0, sizeof g_active[slot]);
    g_active[slot].cinfo = cinfo;                        /* reserved from here on */
  }
  const int no_device = g_no_device;
  pthread_mutex_unlock(&g_lock);
  if (slot < 0) { *why = "too many concurrent compressors"; return -1; }
  if (!enc && !no_device) {
    if (b200jpeg_encoder_create(&enc, 0) != B200JPEG_OK) { enc = NULL; pthread_mutex_lock(&g_lock); g_no_device = 1; pthread_mutex_unlock(&g_lock); }
  }
  if (!enc) {
    pthread_mutex_lock(&g_lock); memset(&g_active[slot], 0, sizeof g_active[slot]); pthread_mutex_unlock(&g_lock);
    *why = b200jpeg_last_error(); return -1;
  }
  g_active[slot].enc = enc;
  return slot;
}

/* the data unit initial_setup sizes components in: a block, or one sample in lossless mode (jcmaster.c:171) */
static int data_unit(j_compress_ptr cinfo) { return cinfo->master->lossless ? 1 : DCTSIZE; }

/* width_in_blocks / height_in_blocks as initial_setup computes them (jcmaster.c:215-242); the reference's master
 * control is not run on objects that take the device path, so they are derived here */
static void comp_blocks(j_compress_ptr cinfo, int ci, JDIMENSION *wib, JDIMENSION *hib)
{
  int hmax = 1, vmax = 1;
  const int du = data_unit(cinfo);
  for (int k = 0; k < cinfo->num_components; k++) { if (cinfo->comp_info[k].h_samp_factor > hmax) hmax = cinfo->comp_info[k].h_samp_factor; if (cinfo->comp_info[k].v_samp_factor > vmax) vmax = cinfo->comp_info[k].v_samp_factor; }
  *wib = (JDIMENSION)(((long)cinfo->image_width * cinfo->comp_info[ci].h_samp_factor + hmax * du - 1) / (hmax * du));
  *hib = (JDIMENSION)(((long)cinfo->image_height * cinfo->comp_info[ci].v_samp_factor + vmax * du - 1) / (vmax * du));
}

/* The derived fields initial_setup (jcmaster.c:209-257) leaves in the object: applications read them after
 * jpeg_start_compress / jpeg_write_coefficients (jpegtran's transforms loop over comp_info[].width_in_blocks and use
 * max_h_samp_factor, jtransform_execute_transformation), so the device path fills them in too. */
static void derive_geometry(j_compress_ptr cinfo)
{
  cinfo->max_h_samp_factor = 1; cinfo->max_v_samp_factor = 1;
  for (int ci = 0; ci < cinfo->num_components; ci++) {
    if (cinfo->comp_info[ci].h_samp_factor > cinfo->max_h_samp_factor) cinfo->max_h_samp_factor = cinfo->comp_info[ci].h_samp_factor;
    if (cinfo->comp_info[ci].v_samp_factor > cinfo->max_v_samp_factor) cinfo->max_v_samp_factor = cinfo->comp_info[ci].v_samp_factor;
  }
  for (int ci = 0; ci < cinfo->num_components; ci++) {
    jpeg_component_info *c = &cinfo->comp_info[ci];
    c->component_index = ci;
    c->DCT_scaled_size = data_unit(cinfo);
    comp_blocks(cinfo, ci, &c->width_in_blocks, &c->height_in_blocks);
    c->downsampled_width = (JDIMENSION)(((long)cinfo->image_width * c->h_samp_factor + cinfo->max_h_samp_factor - 1) / cinfo->max_h_samp_factor);
    c->downsampled_height = (JDIMENSION)(((long)cinfo->image_height * c->v_samp_factor + cinfo->max_v_samp_factor - 1) / cinfo->max_v_samp_factor);
    c->component_needed = TRUE;
  }
  const long rows = (long)cinfo->max_v_samp_factor * data_unit(cinfo);
  cinfo->total_iMCU_rows = (JDIMENSION)(((long)cinfo->image_height + rows - 1) / rows);
}

/* jinit_c_master_control's lossless decisions (jcmaster.c:1055-1094), made on the object before its parameters are
 * read.  A script decides lossless mode by its first entry (validate_script, jcmaster.c:301-329), except the scan
 * search's script, which is not validated; without a script jpeg_enable_lossless has decided it.  Lossless mode then
 * overrides smoothing, the colour space, subsampling and raw-data input, and forces optimal Huffman tables.  The
 * reference makes the same changes when it runs instead, so an object it gets back is already in the state it would
 * put it in. */
static void lossless_overrides(j_compress_ptr cinfo)
{
  if (cinfo->scan_info != NULL && cinfo->num_scans > 0 && !cinfo->master->optimize_scans)
    cinfo->master->lossless = cinfo->scan_info[0].Ss != 0 && cinfo->scan_info[0].Se == 0;
  if (!cinfo->master->lossless) return;
  cinfo->raw_data_in = FALSE;
  cinfo->smoothing_factor = 0;
  jpeg_default_colorspace(cinfo);
  for (int ci = 0; ci < cinfo->num_components; ci++) cinfo->comp_info[ci].h_samp_factor = cinfo->comp_info[ci].v_samp_factor = 1;
  if (!cinfo->arith_code) cinfo->optimize_coding = TRUE;
}

/* the encoder-relevant state of the reference's object -> b200jpeg_params.  Returns 0 if the
 * object uses something the parameter block cannot express (then the reference encodes it). */
static int fill_params(j_compress_ptr cinfo, boolean write_all_tables, b200jpeg_params *p)
{
  int i, ci;
  memset(p, 0, sizeof(*p));
  if (!write_all_tables) return 0;                       /* abbreviated datastreams: reference only */
  const int lossless = cinfo->master->lossless;
  if ((cinfo->data_precision != 8 && cinfo->data_precision != 12 && !(lossless && cinfo->data_precision == 16)) || cinfo->arith_code) return 0;
  if (cinfo->data_precision == 12 && cinfo->raw_data_in) return 0;   /* jpeg12_write_raw_data: reference only */
  if (lossless && cinfo->scan_info != NULL && cinfo->num_scans <= 0) return 0;   /* the reference refuses the empty script */
  if (cinfo->num_components > B200JPEG_MAX_COMPONENTS || cinfo->num_scans > B200JPEG_MAX_SCANS) return 0;
  switch (cinfo->in_color_space) {
  case JCS_GRAYSCALE: p->in_color_space = B200JPEG_CS_GRAYSCALE; break;
  case JCS_RGB: case JCS_EXT_RGB: p->in_color_space = B200JPEG_CS_RGB; break;
  case JCS_YCbCr: p->in_color_space = B200JPEG_CS_YCbCr; break;
  case JCS_CMYK: p->in_color_space = B200JPEG_CS_CMYK; break;
  case JCS_YCCK: p->in_color_space = B200JPEG_CS_YCCK; break;
  case JCS_UNKNOWN: p->in_color_space = B200JPEG_CS_UNKNOWN; break;
  /* the other pixel orders of the RGB family (jccolor.c:253-291): same numeric values as J_COLOR_SPACE */
  case JCS_EXT_RGBX: case JCS_EXT_BGR: case JCS_EXT_BGRX: case JCS_EXT_XBGR: case JCS_EXT_XRGB:
  case JCS_EXT_RGBA: case JCS_EXT_BGRA: case JCS_EXT_ABGR: case JCS_EXT_ARGB:
    p->in_color_space = (int)cinfo->in_color_space; break;
  default: return 0;
  }
  switch (cinfo->jpeg_color_space) {
  case JCS_GRAYSCALE: p->jpeg_color_space = B200JPEG_CS_GRAYSCALE; break;
  case JCS_YCbCr: p->jpeg_color_space = B200JPEG_CS_YCbCr; break;
  case JCS_RGB: p->jpeg_color_space = B200JPEG_CS_RGB; break;
  case JCS_CMYK: p->jpeg_color_space = B200JPEG_CS_CMYK; break;
  case JCS_YCCK: p->jpeg_color_space = B200JPEG_CS_YCCK; break;
  case JCS_UNKNOWN: p->jpeg_color_space = B200JPEG_CS_UNKNOWN; break;
  default: return 0;
  }
  p->image_width = (int)cinfo->image_width;   p->image_height = (int)cinfo->image_height;
  p->input_components = cinfo->input_components;
  p->data_precision = cinfo->data_precision;
  p->num_components = cinfo->num_components;
  for (ci = 0; ci < cinfo->num_components; ci++) {
    jpeg_component_info *c = &cinfo->comp_info[ci];
    p->comp_info[ci].component_id = c->component_id;
    p->comp_info[ci].h_samp_factor = c->h_samp_factor;  p->comp_info[ci].v_samp_factor = c->v_samp_factor;
    p->comp_info[ci].quant_tbl_no = c->quant_tbl_no;
    p->comp_info[ci].dc_tbl_no = c->dc_tbl_no;          p->comp_info[ci].ac_tbl_no = c->ac_tbl_no;
  }
  for (i = 0; i < NUM_QUANT_TBLS; i++) if (cinfo->quant_tbl_ptrs[i]) {
    for (int k = 0; k < DCTSIZE2; k++) p->quant_tbl[i][k] = cinfo->quant_tbl_ptrs[i]->quantval[k];
    p->quant_tbl_present[i] = 1;
  }
  for (i = 0; i < NUM_HUFF_TBLS; i++) {
    if (cinfo->dc_huff_tbl_ptrs[i]) { memcpy(p->dc_huff_tbl[i].bits, cinfo->dc_huff_tbl_ptrs[i]->bits, 17);
      memcpy(p->dc_huff_tbl[i].huffval, cinfo->dc_huff_tbl_ptrs[i]->huffval, 256); p->dc_huff_tbl[i].present = 1; }
    if (cinfo->ac_huff_tbl_ptrs[i]) { memcpy(p->ac_huff_tbl[i].bits, cinfo->ac_huff_tbl_ptrs[i]->bits, 17);
      memcpy(p->ac_huff_tbl[i].huffval, cinfo->ac_huff_tbl_ptrs[i]->huffval, 256); p->ac_huff_tbl[i].present = 1; }
  }
  p->num_scans = cinfo->scan_info ? cinfo->num_scans : 0;
  for (i = 0; i < p->num_scans; i++) {
    p->scan_info[i].comps_in_scan = cinfo->scan_info[i].comps_in_scan;
    for (int k = 0; k < MAX_COMPS_IN_SCAN; k++) p->scan_info[i].component_index[k] = cinfo->scan_info[i].component_index[k];
    p->scan_info[i].Ss = cinfo->scan_info[i].Ss; p->scan_info[i].Se = cinfo->scan_info[i].Se;
    p->scan_info[i].Ah = cinfo->scan_info[i].Ah; p->scan_info[i].Al = cinfo->scan_info[i].Al;
  }
  p->optimize_coding = cinfo->optimize_coding;   p->dct_method = cinfo->dct_method;
  p->restart_interval = (int)cinfo->restart_interval; p->restart_in_rows = cinfo->restart_in_rows;
  p->smoothing_factor = cinfo->smoothing_factor;
  p->write_JFIF_header = cinfo->write_JFIF_header; p->write_Adobe_marker = cinfo->write_Adobe_marker;
  p->JFIF_major_version = cinfo->JFIF_major_version; p->JFIF_minor_version = cinfo->JFIF_minor_version;
  p->density_unit = cinfo->density_unit; p->X_density = cinfo->X_density; p->Y_density = cinfo->Y_density;
  /* mozjpeg extension block, jpegint.h:93-135 */
  p->compress_profile = cinfo->master->compress_profile;  p->optimize_scans = cinfo->master->optimize_scans;
  p->trellis_quant = cinfo->master->trellis_quant;        p->trellis_quant_dc = cinfo->master->trellis_quant_dc;
  p->trellis_eob_opt = cinfo->master->trellis_eob_opt;    p->use_scans_in_trellis = cinfo->master->use_scans_in_trellis;
  p->trellis_q_opt = cinfo->master->trellis_q_opt;        p->overshoot_deringing = cinfo->master->overshoot_deringing;
  p->trellis_freq_split = cinfo->master->trellis_freq_split; p->trellis_num_loops = cinfo->master->trellis_num_loops;
  p->lambda_log_scale1 = cinfo->master->lambda_log_scale1; p->lambda_log_scale2 = cinfo->master->lambda_log_scale2;
  p->trellis_delta_dc_weight = cinfo->master->trellis_delta_dc_weight;
  p->use_lambda_weight_tbl = cinfo->master->use_lambda_weight_tbl;
  p->quant_tbl_master_idx = cinfo->master->quant_tbl_master_idx; p->dc_scan_opt_mode = cinfo->master->dc_scan_opt_mode;
  return 1;
}

/* jpeg_enable_lossless keeps its predictor and point transform in cinfo->Ss / Al and leaves scan_info alone: the block
 * gets the same call.  Beside the scan search's script the C-ABI refuses it (the reference writes SOF2 headers there).
 * A script that is itself lossless is in the block already. */
static const char *finish_lossless_params(j_compress_ptr cinfo, b200jpeg_params *p)
{
  if (!cinfo->master->lossless || (cinfo->scan_info != NULL && !cinfo->master->optimize_scans)) return NULL;
  return b200jpeg_enable_lossless(p, cinfo->Ss, cinfo->Al) == B200JPEG_OK ? NULL : b200jpeg_last_error();
}

/* 16-bit samples (J16SAMPLE = unsigned short, lossless mode only).  jpeg16_write_scanlines is not taken over: the
 * reference's own (jcapistd.c:90-135 compiled with BITS_IN_JSAMPLE 16) checks precision and state, calls the progress
 * monitor, drops rows past the bottom of the image and hands the rest to the main controller's process_data_16
 * (jcapistd.c:126-129).  jpeg_start_compress installs this function there for 16-bit device-path objects, so the rows
 * go to b200jpeg_write_scanlines as uint16 rows; the reference advances next_scanline by what it reports. */
static void device_process_data_16(j_compress_ptr cinfo, J16SAMPARRAY rows, JDIMENSION *row_ctr, JDIMENSION rows_avail)
{
  int slot = find_active(cinfo);
  if (slot < 0) ERREXIT1(cinfo, JERR_BAD_STATE, cinfo->global_state);
  if (rows_avail == 0) return;
  int took = b200jpeg_write_scanlines(g_active[slot].enc, (const uint8_t *const *)rows, (int)rows_avail);
  if (took < 0) ERREXIT1(cinfo, JERR_BAD_STATE, cinfo->global_state);
  *row_ctr += (JDIMENSION)took;
}

GLOBAL(void)
jpeg_start_compress(j_compress_ptr cinfo, boolean write_all_tables)
{
  static start_fn real;
  if (!real) real = (start_fn)next_sym("jpeg_start_compress");
  b200jpeg_params p;
  const char *why = NULL;
  int slot = -1;
  if (cinfo->global_state != CSTATE_START) { real(cinfo, write_all_tables); return; }   /* let the reference raise JERR_BAD_STATE */
  if (getenv("MOZ_B200_FORCE_CPU")) why = "MOZ_B200_FORCE_CPU is set";
  /* jcapistd.c:53-56 */
  if (cinfo->master->num_scans_luma == 0 || cinfo->scan_info == NULL || cinfo->num_scans == 0)
    cinfo->master->optimize_scans = FALSE;
  if (!why) lossless_overrides(cinfo);
  if (!why && !fill_params(cinfo, write_all_tables, &p)) why = "parameter set outside b200jpeg_params";
  if (!why) why = finish_lossless_params(cinfo, &p);
  if (!why && b200jpeg_validate(&p) != B200JPEG_OK) why = b200jpeg_last_error();
  if (!why) slot = claim_slot(cinfo, &why);
  if (!why && !cinfo->raw_data_in) {
    /* raw-data objects (jpeg_write_raw_data) collect their planes on the host and encode at finish time */
    if (b200jpeg_start_compress(g_active[slot].enc, &p) != B200JPEG_OK) { why = b200jpeg_last_error(); release_slot(slot); slot = -1; }
  }
  if (why) {
    if (verbose()) fprintf(stderr, "b200 shim: reference path (%s)\n", why);
    if (required()) { fprintf(stderr, "b200 shim: B200_SHIM_REQUIRE=1 and the device path was not taken: %s\n", why); ERREXIT(cinfo, JERR_NOTIMPL); }
    real(cinfo, write_all_tables);
    return;
  }
  if (verbose()) fprintf(stderr, "b200 shim: device path (%s%ux%u, %d scans)\n", cinfo->raw_data_in ? "raw data, " : cinfo->master->lossless ? "lossless, " : "",
                         cinfo->image_width, cinfo->image_height, p.num_scans);
  g_active[slot].header_len = 2 + (p.write_JFIF_header ? 18 : 0) + (p.write_Adobe_marker ? 16 : 0);
  g_active[slot].total_passes = b200jpeg_total_passes(&p);
  g_active[slot].lossless = cinfo->master->lossless;
  if (cinfo->progress != NULL) { cinfo->progress->completed_passes = 0; cinfo->progress->total_passes = g_active[slot].total_passes; }   /* prepare_for_pass, jcmaster.c:711-714 */
  if (cinfo->raw_data_in) {
    g_active[slot].raw = 1; g_active[slot].params = p;
    for (int ci = 0; ci < cinfo->num_components; ci++) {
      JDIMENSION wib, hib; comp_blocks(cinfo, ci, &wib, &hib);
      g_active[slot].plane_pitch[ci] = (size_t)wib * DCTSIZE; g_active[slot].plane_rows[ci] = (size_t)hib * DCTSIZE;
      g_active[slot].plane[ci] = (uint8_t *)calloc(g_active[slot].plane_pitch[ci], g_active[slot].plane_rows[ci]);
      if (!g_active[slot].plane[ci]) { release_slot(slot); ERREXIT1(cinfo, JERR_OUT_OF_MEMORY, 0); }
    }
  }
  if (cinfo->data_precision == 16) {
    /* the main controller jinit_c_main_controller would have made, reduced to what jpeg16_write_scanlines calls; in the
     * image pool like the reference's, so jpeg_abort frees it */
    struct jpeg_c_main_controller *m = (struct jpeg_c_main_controller *)(*cinfo->mem->alloc_small) ((j_common_ptr)cinfo, JPOOL_IMAGE, sizeof *m);
    memset(m, 0, sizeof *m);
    m->process_data_16 = device_process_data_16;
    cinfo->main = m;
    cinfo->master->call_pass_startup = FALSE;                       /* the headers are the device's (jcapistd.c:117-118) */
  }
  derive_geometry(cinfo);
  jpeg_suppress_tables(cinfo, FALSE);                               /* jcapistd.c:50-51 (write_all_tables is TRUE here) */
  (*cinfo->err->reset_error_mgr) ((j_common_ptr)cinfo);
  cinfo->next_scanline = 0;
  cinfo->global_state = cinfo->raw_data_in ? CSTATE_RAW_OK : CSTATE_SCANNING;
}

/* jpeg_write_raw_data (jcapistd.c:145-195): one iMCU row of already converted, downsampled component rows per call;
 * compress_first_pass (jccoefct.c:262-353) reads v_samp_factor*8 rows of width_in_blocks*8 samples of every component */
typedef JDIMENSION (*rawdata_fn)(j_compress_ptr, JSAMPIMAGE, JDIMENSION);
GLOBAL(JDIMENSION)
jpeg_write_raw_data(j_compress_ptr cinfo, JSAMPIMAGE data, JDIMENSION num_lines)
{
  static rawdata_fn real;
  int slot = find_active(cinfo);
  if (slot < 0) { if (!real) real = (rawdata_fn)next_sym("jpeg_write_raw_data"); return real(cinfo, data, num_lines); }
  if (cinfo->global_state != CSTATE_RAW_OK || !g_active[slot].raw) ERREXIT1(cinfo, JERR_BAD_STATE, cinfo->global_state);
  if (cinfo->next_scanline >= cinfo->image_height) { WARNMS(cinfo, JWRN_TOO_MUCH_DATA); return 0; }
  if (cinfo->progress != NULL) {
    cinfo->progress->pass_counter = (long)cinfo->next_scanline;
    cinfo->progress->pass_limit = (long)cinfo->image_height;
    (*cinfo->progress->progress_monitor) ((j_common_ptr)cinfo);
  }
  int vmax = 1;
  for (int k = 0; k < cinfo->num_components; k++) if (cinfo->comp_info[k].v_samp_factor > vmax) vmax = cinfo->comp_info[k].v_samp_factor;
  const JDIMENSION lines_per_iMCU_row = (JDIMENSION)(vmax * DCTSIZE);
  if (num_lines < lines_per_iMCU_row) ERREXIT(cinfo, JERR_BUFFER_SIZE);
  const size_t imcu = cinfo->next_scanline / lines_per_iMCU_row;
  for (int ci = 0; ci < cinfo->num_components; ci++) {
    const size_t rows = (size_t)cinfo->comp_info[ci].v_samp_factor * DCTSIZE, r0 = imcu * rows;
    for (size_t r = 0; r < rows && r0 + r < g_active[slot].plane_rows[ci]; r++)
      memcpy(g_active[slot].plane[ci] + (r0 + r) * g_active[slot].plane_pitch[ci], data[ci][r], g_active[slot].plane_pitch[ci]);
  }
  cinfo->next_scanline += lines_per_iMCU_row;
  return lines_per_iMCU_row;
}

static JDIMENSION device_write_scanlines(j_compress_ptr cinfo, int slot, const uint8_t *const *rows, JDIMENSION num_lines, int precision)
{
  if (cinfo->data_precision != precision) ERREXIT1(cinfo, JERR_BAD_PRECISION, cinfo->data_precision);   /* jcapistd.c:97-98 */
  if (cinfo->global_state != CSTATE_SCANNING) ERREXIT1(cinfo, JERR_BAD_STATE, cinfo->global_state);
  if (cinfo->next_scanline >= cinfo->image_height) WARNMS(cinfo, JWRN_TOO_MUCH_DATA);   /* jcapistd.c:103-104 */
  if (cinfo->progress != NULL) {                                                         /* jcapistd.c:107-111 */
    cinfo->progress->pass_counter = (long)cinfo->next_scanline;
    cinfo->progress->pass_limit = (long)cinfo->image_height;
    (*cinfo->progress->progress_monitor) ((j_common_ptr)cinfo);
  }
  int took = b200jpeg_write_scanlines(g_active[slot].enc, rows, (int)num_lines);
  if (took < 0) ERREXIT1(cinfo, JERR_BAD_STATE, cinfo->global_state);
  cinfo->next_scanline += (JDIMENSION)took;
  return (JDIMENSION)took;
}

GLOBAL(JDIMENSION)
jpeg_write_scanlines(j_compress_ptr cinfo, JSAMPARRAY scanlines, JDIMENSION num_lines)
{
  static write_fn real;
  int slot = find_active(cinfo);
  if (slot < 0) { if (!real) real = (write_fn)next_sym("jpeg_write_scanlines"); return real(cinfo, scanlines, num_lines); }
  return device_write_scanlines(cinfo, slot, (const uint8_t *const *)scanlines, num_lines, 8);
}

/* 12-bit samples (J12SAMPLE = short): same entry point, rows of uint16 (jcapistd.c compiled with BITS_IN_JSAMPLE 12) */
typedef JDIMENSION (*write12_fn)(j_compress_ptr, J12SAMPARRAY, JDIMENSION);
GLOBAL(JDIMENSION)
jpeg12_write_scanlines(j_compress_ptr cinfo, J12SAMPARRAY scanlines, JDIMENSION num_lines)
{
  static write12_fn real;
  int slot = find_active(cinfo);
  if (slot < 0) { if (!real) real = (write12_fn)next_sym("jpeg12_write_scanlines"); return real(cinfo, scanlines, num_lines); }
  return device_write_scanlines(cinfo, slot, (const uint8_t *const *)scanlines, num_lines, 12);
}

/* hand the finished datastream to the application's destination manager (jpeglib.h:897-904) */
static void push_bytes(j_compress_ptr cinfo, int slot, const uint8_t *src, size_t n)
{
  size_t off = 0;
  while (off < n) {
    size_t k = n - off < cinfo->dest->free_in_buffer ? n - off : cinfo->dest->free_in_buffer;
    memcpy(cinfo->dest->next_output_byte, src + off, k);
    cinfo->dest->next_output_byte += k; cinfo->dest->free_in_buffer -= k; off += k;
    if (cinfo->dest->free_in_buffer == 0) {
      if (!(*cinfo->dest->empty_output_buffer) (cinfo)) { release_slot(slot); ERREXIT(cinfo, JERR_CANT_SUSPEND); }
    }
  }
}

/* the caller's coefficient arrays -> one contiguous plane per component -> b200jpeg_encode_batch_coefs */
static int encode_coef_arrays(j_compress_ptr cinfo, int slot)
{
  b200jpeg_params *p = &g_active[slot].params;
  const int16_t *planes[4] = {NULL, NULL, NULL, NULL}; size_t pitch[4] = {0, 0, 0, 0}, stride[4] = {0, 0, 0, 0};
  int16_t *buf[4] = {NULL, NULL, NULL, NULL};
  int rc = B200JPEG_OK;
  for (int ci = 0; ci < cinfo->num_components; ci++) {
    JDIMENSION wib, hib; comp_blocks(cinfo, ci, &wib, &hib);
    buf[ci] = (int16_t *)malloc((size_t)wib * hib * DCTSIZE2 * sizeof(int16_t));
    if (!buf[ci]) { rc = B200JPEG_ERR_BUFFER; break; }
    for (JDIMENSION r = 0; r < hib; r++) {
      JBLOCKARRAY rows = (*cinfo->mem->access_virt_barray) ((j_common_ptr)cinfo, g_active[slot].coef_arrays[ci], r, 1, FALSE);
      memcpy(buf[ci] + (size_t)r * wib * DCTSIZE2, rows[0], (size_t)wib * DCTSIZE2 * sizeof(JCOEF));
    }
    planes[ci] = buf[ci]; pitch[ci] = wib; stride[ci] = (size_t)wib * hib;
  }
  if (rc == B200JPEG_OK) rc = b200jpeg_encode_batch_coefs(g_active[slot].enc, p, planes, 0, pitch, stride, 1);
  for (int ci = 0; ci < 4; ci++) free(buf[ci]);
  return rc;
}

GLOBAL(void)
jpeg_finish_compress(j_compress_ptr cinfo)
{
  static finish_fn real;
  int slot = find_active(cinfo);
  if (slot < 0) { if (!real) real = (finish_fn)next_sym("jpeg_finish_compress"); real(cinfo); return; }
  const int from_coefs = g_active[slot].coef_arrays != NULL;
  if (!from_coefs && cinfo->next_scanline < cinfo->image_height) { release_slot(slot); ERREXIT(cinfo, JERR_TOO_LITTLE_DATA); }   /* jcapimin.c:183-184 */
  const uint8_t *jpg; size_t n;
  b200jpeg_encoder *enc = g_active[slot].enc;
  int rc;                                                            /* all device work happens here, on the caller's thread */
  if (from_coefs) { rc = encode_coef_arrays(cinfo, slot); if (rc == B200JPEG_OK) rc = b200jpeg_get_output(enc, 0, &jpg, &n); }
  else if (g_active[slot].raw) {
    size_t stride[4];
    for (int ci = 0; ci < 4; ci++) stride[ci] = g_active[slot].plane_pitch[ci] * g_active[slot].plane_rows[ci];
    rc = b200jpeg_encode_batch_raw(enc, &g_active[slot].params, (const uint8_t *const *)g_active[slot].plane, 0, g_active[slot].plane_pitch, stride, 1);
    if (rc == B200JPEG_OK) rc = b200jpeg_get_output(enc, 0, &jpg, &n);
  }
  else rc = b200jpeg_finish_compress(enc, &jpg, &n);
  if (rc != B200JPEG_OK) {
    release_slot(slot);
    fprintf(stderr, "b200 shim: %s\n", b200jpeg_last_error());
    if (rc == B200JPEG_ERR_BAD_DCT_COEF) ERREXIT(cinfo, JERR_BAD_DCT_COEF);
    ERREXIT(cinfo, JERR_NOTIMPL);
  }
  /* the remaining passes ran inside the one device call; the application's monitor hears about each of them, on this
   * thread, with the counters the reference's loop would show at the end of the pass (jcapimin.c:193-215,
   * jcmaster.c:711-714).  Lossless objects hear every row of the reference's loop, as they did when the reference
   * encoded them. */
  if (cinfo->progress != NULL) {
    const int tp = g_active[slot].total_passes;
    const long rows = (long)cinfo->total_iMCU_rows;
    const long first = g_active[slot].lossless ? 0 : rows, last = g_active[slot].lossless ? rows - 1 : rows;
    for (int pass = from_coefs ? 0 : 1; pass < tp; pass++) {
      for (long r = first; r <= last; r++) {
        cinfo->progress->completed_passes = pass; cinfo->progress->total_passes = tp;
        cinfo->progress->pass_counter = r; cinfo->progress->pass_limit = rows;
        (*cinfo->progress->progress_monitor) ((j_common_ptr)cinfo);
      }
    }
  }
  if (!from_coefs) (*cinfo->dest->init_destination) (cinfo);         /* jpeg_write_coefficients did it already (jctrans.c:57) */
  /* the file header, the application's own marker segments (written right behind it, like the reference's marker
   * writer would have), then the rest */
  size_t hl = g_active[slot].header_len < n ? g_active[slot].header_len : n;
  push_bytes(cinfo, slot, jpg, hl);
  if (g_active[slot].extra_len) push_bytes(cinfo, slot, g_active[slot].extra, g_active[slot].extra_len);
  push_bytes(cinfo, slot, jpg + hl, n - hl);
  (*cinfo->dest->term_destination) (cinfo);
  /* tables are now "sent" (jcmarker.c sets sent_table as it writes them) */
  for (int i = 0; i < NUM_QUANT_TBLS; i++) if (cinfo->quant_tbl_ptrs[i]) cinfo->quant_tbl_ptrs[i]->sent_table = TRUE;
  for (int i = 0; i < NUM_HUFF_TBLS; i++) {
    if (cinfo->dc_huff_tbl_ptrs[i]) cinfo->dc_huff_tbl_ptrs[i]->sent_table = TRUE;
    if (cinfo->ac_huff_tbl_ptrs[i]) cinfo->ac_huff_tbl_ptrs[i]->sent_table = TRUE;
  }
  release_slot_ex(slot, 1);
  jpeg_abort((j_common_ptr)cinfo);                                   /* back to CSTATE_START (jcapimin.c:227) */
}

/* jpeg_write_coefficients (jctrans.c:39-66): the arrays may still be empty here (jpegtran fills them afterwards,
 * jtransform_execute_transformation), so they are only remembered; jpeg_finish_compress reads and encodes them. */
typedef void (*wrcoef_fn)(j_compress_ptr, jvirt_barray_ptr *);
GLOBAL(void)
jpeg_write_coefficients(j_compress_ptr cinfo, jvirt_barray_ptr *coef_arrays)
{
  static wrcoef_fn real;
  if (!real) real = (wrcoef_fn)next_sym("jpeg_write_coefficients");
  b200jpeg_params p;
  const char *why = NULL;
  int slot = -1;
  if (cinfo->global_state != CSTATE_START || cinfo->master->lossless) { real(cinfo, coef_arrays); return; }   /* the reference raises the error */
  if (getenv("MOZ_B200_FORCE_CPU")) why = "MOZ_B200_FORCE_CPU is set";
  if (cinfo->master->num_scans_luma == 0) cinfo->master->optimize_scans = FALSE;        /* jctrans.c:49-50 */
  if (!why && !fill_params(cinfo, TRUE, &p)) why = "parameter set outside b200jpeg_params";
  if (!why) {
    /* no pixels on this path: the input colour space of the object (whatever jpeg_copy_critical_parameters and the
     * application left there, e.g. YCbCr after jpegtran -grayscale) has no meaning, as in transencode_master_selection
     * (jctrans.c:181-184) */
    p.in_color_space = p.jpeg_color_space; p.input_components = p.num_components;
  }
  if (!why && p.trellis_quant) why = "trellis quantization requested on coefficient input";
  if (!why && b200jpeg_validate(&p) != B200JPEG_OK) why = b200jpeg_last_error();
  if (!why) slot = claim_slot(cinfo, &why);
  if (why) {
    if (verbose()) fprintf(stderr, "b200 shim: reference path (%s)\n", why);
    if (required()) { fprintf(stderr, "b200 shim: B200_SHIM_REQUIRE=1 and the device path was not taken: %s\n", why); ERREXIT(cinfo, JERR_NOTIMPL); }
    real(cinfo, coef_arrays);
    return;
  }
  if (verbose()) fprintf(stderr, "b200 shim: device path (coefficients, %ux%u, %d scans)\n", cinfo->image_width, cinfo->image_height, p.num_scans);
  g_active[slot].coef_arrays = coef_arrays; g_active[slot].params = p;
  g_active[slot].total_passes = b200jpeg_total_passes(&p);
  if (cinfo->progress != NULL) { cinfo->progress->completed_passes = 0; cinfo->progress->total_passes = g_active[slot].total_passes; }
  g_active[slot].header_len = 2 + (p.write_JFIF_header ? 18 : 0) + (p.write_Adobe_marker ? 16 : 0);
  derive_geometry(cinfo);
  jpeg_suppress_tables(cinfo, FALSE);                                /* jctrans.c:54 */
  (*cinfo->err->reset_error_mgr) ((j_common_ptr)cinfo);
  (*cinfo->dest->init_destination) (cinfo);
  (*cinfo->mem->realize_virt_arrays) ((j_common_ptr)cinfo);          /* arrays requested from this object's pool (jctrans.c:211) */
  cinfo->next_scanline = 0;                                          /* so jpeg_write_marker works (jctrans.c:63) */
  cinfo->global_state = CSTATE_WRCOEFS;
}

/* an application that gives up mid-image: through the compress-specific entry points or the generic ones
 * (jpeg_abort / jpeg_destroy, jcomapi.c:29-98, which jpeg_abort_compress / jpeg_destroy_compress forward to) */
static void drop_object(void *cinfo)
{
  int slot = find_active((j_compress_ptr)cinfo);
  if (slot >= 0) release_slot(slot);
}
GLOBAL(void)
jpeg_abort_compress(j_compress_ptr cinfo)
{
  static abort_fn real;
  drop_object(cinfo);
  if (!real) real = (abort_fn)next_sym("jpeg_abort_compress");
  real(cinfo);
}
GLOBAL(void)
jpeg_destroy_compress(j_compress_ptr cinfo)
{
  static abort_fn real;
  drop_object(cinfo);
  if (!real) real = (abort_fn)next_sym("jpeg_destroy_compress");
  real(cinfo);
}
typedef void (*common_fn)(j_common_ptr);
GLOBAL(void)
jpeg_abort(j_common_ptr cinfo)
{
  static common_fn real;
  if (!cinfo->is_decompressor) drop_object(cinfo);
  if (!real) real = (common_fn)next_sym("jpeg_abort");
  real(cinfo);
}
GLOBAL(void)
jpeg_destroy(j_common_ptr cinfo)
{
  static common_fn real;
  if (!cinfo->is_decompressor) drop_object(cinfo);
  if (!real) real = (common_fn)next_sym("jpeg_destroy");
  real(cinfo);
}

/* Marker segments an application writes between jpeg_start_compress / jpeg_write_coefficients and the first
 * data (jpeg_write_marker, jpeg_write_m_header + jpeg_write_m_byte, jcapimin.c:232-290): the reference's marker writer
 * would put them right behind the file header; the device path keeps them and splices them in at the same place. */
static void extra_put(int slot, j_compress_ptr cinfo, const unsigned char *d, size_t n)
{
  if (g_active[slot].extra_len + n > g_active[slot].extra_cap) {
    size_t cap = g_active[slot].extra_cap ? g_active[slot].extra_cap * 2 : 4096;
    while (cap < g_active[slot].extra_len + n) cap *= 2;
    unsigned char *q = (unsigned char *)realloc(g_active[slot].extra, cap);
    if (!q) ERREXIT1(cinfo, JERR_OUT_OF_MEMORY, 0);
    g_active[slot].extra = q; g_active[slot].extra_cap = cap;
  }
  memcpy(g_active[slot].extra + g_active[slot].extra_len, d, n); g_active[slot].extra_len += n;
}
static void marker_state_check(j_compress_ptr cinfo)
{
  if (cinfo->next_scanline != 0 || (cinfo->global_state != CSTATE_SCANNING && cinfo->global_state != CSTATE_RAW_OK && cinfo->global_state != CSTATE_WRCOEFS))
    ERREXIT1(cinfo, JERR_BAD_STATE, cinfo->global_state);
}
GLOBAL(void)
jpeg_write_marker(j_compress_ptr cinfo, int marker, const JOCTET *dataptr, unsigned int datalen)
{
  static marker_fn real;
  int slot = find_active(cinfo);
  if (slot >= 0) {
    marker_state_check(cinfo);
    if (datalen > 65533u) ERREXIT(cinfo, JERR_BAD_LENGTH);           /* write_marker_header, jcmarker.c:609-619 */
    unsigned char h[4] = {0xFF, (unsigned char)marker, (unsigned char)((datalen + 2) >> 8), (unsigned char)((datalen + 2) & 0xFF)};
    extra_put(slot, cinfo, h, 4);
    extra_put(slot, cinfo, dataptr, datalen);
    return;
  }
  if (!real) real = (marker_fn)next_sym("jpeg_write_marker");
  real(cinfo, marker, dataptr, datalen);
}
typedef void (*mheader_fn)(j_compress_ptr, int, unsigned int);
typedef void (*mbyte_fn)(j_compress_ptr, int);
GLOBAL(void)
jpeg_write_m_header(j_compress_ptr cinfo, int marker, unsigned int datalen)
{
  static mheader_fn real;
  int slot = find_active(cinfo);
  if (slot >= 0) {
    marker_state_check(cinfo);
    if (datalen > 65533u) ERREXIT(cinfo, JERR_BAD_LENGTH);
    unsigned char h[4] = {0xFF, (unsigned char)marker, (unsigned char)((datalen + 2) >> 8), (unsigned char)((datalen + 2) & 0xFF)};
    extra_put(slot, cinfo, h, 4);
    return;
  }
  if (!real) real = (mheader_fn)next_sym("jpeg_write_m_header");
  real(cinfo, marker, datalen);
}
GLOBAL(void)
jpeg_write_m_byte(j_compress_ptr cinfo, int val)
{
  static mbyte_fn real;
  int slot = find_active(cinfo);
  if (slot >= 0) { unsigned char b = (unsigned char)val; extra_put(slot, cinfo, &b, 1); return; }
  if (!real) real = (mbyte_fn)next_sym("jpeg_write_m_byte");
  real(cinfo, val);
}

#ifndef B200_SHIM_STANDALONE
/*
 * TurboJPEG YUV encoding: tj3EncodeYUVPlanes8 (turbojpeg.c:1467-1619) and tj3EncodeYUV8 (turbojpeg.c:1647-1690) run
 * through b200jpeg_encode_yuv_batch.  The parameter block is what setCompDefaults (turbojpeg.c:330-397) builds from the
 * handle's settings (read with tj3Get).  Bottom-up rows, lossless mode, anything the reference would refuse (so that
 * its error text and tj3GetErrorStr stay its own), MOZ_B200_FORCE_CPU, a host without a device and any refusal of the
 * C-ABI go to the reference's implementation.  (The standalone libjpeg.so.62 carries no TurboJPEG API.)
 */
#include "turbojpeg.h"

typedef int (*tjget_fn)(tjhandle, int);
typedef int (*tjset_fn)(tjhandle, int, int);
typedef int (*tjyuvplanes_fn)(tjhandle, const unsigned char *, int, int, int, int, unsigned char **, int *);
typedef int (*tjyuv8_fn)(tjhandle, const unsigned char *, int, int, int, int, unsigned char *, int);
typedef int (*tjplanedim_fn)(int, int, int);

/* an encoder for one call: the spare one, else a new one (NULL and g_no_device set when there is no device) */
static b200jpeg_encoder *take_encoder(void)
{
  pthread_mutex_lock(&g_lock);
  b200jpeg_encoder *enc = g_idle_enc; g_idle_enc = NULL;
  const int no_device = g_no_device;
  pthread_mutex_unlock(&g_lock);
  if (!enc && !no_device && b200jpeg_encoder_create(&enc, 0) != B200JPEG_OK) {
    enc = NULL; pthread_mutex_lock(&g_lock); g_no_device = 1; pthread_mutex_unlock(&g_lock);
  }
  return enc;
}
static void give_encoder(b200jpeg_encoder *enc)
{
  pthread_mutex_lock(&g_lock);
  if (!g_idle_enc) { g_idle_enc = enc; enc = NULL; }
  pthread_mutex_unlock(&g_lock);
  if (enc) b200jpeg_encoder_destroy(enc);
}

/* the device path of tj3EncodeYUVPlanes8: NULL when the planes are written, else why the reference has to run */
static const char *encode_yuv_device(tjhandle handle, const unsigned char *srcBuf, int width, int pitch, int height,
                                     int pixelFormat, unsigned char **dstPlanes, int *strides)
{
  static tjget_fn get; static tjset_fn set;
  if (!get) get = (tjget_fn)next_sym("tj3Get");
  if (!set) set = (tjset_fn)next_sym("tj3Set");
  if (getenv("MOZ_B200_FORCE_CPU")) return "MOZ_B200_FORCE_CPU is set";
  /* turbojpeg.c:1488-1503 */
  if (!handle || !srcBuf || width <= 0 || pitch < 0 || height <= 0 || pixelFormat < 0 || pixelFormat >= TJ_NUMPF || !dstPlanes || !dstPlanes[0])
    return "an argument the reference refuses";
  /* a compress instance takes TJPARAM_OPTIMIZE, a decompress-only one refuses it: setting the current value tells them
   * apart without changing anything */
  if (set(handle, TJPARAM_OPTIMIZE, get(handle, TJPARAM_OPTIMIZE)) != 0) return "not a compress instance";
  const int subsamp = get(handle, TJPARAM_SUBSAMP);
  if (subsamp < 0 || subsamp >= TJ_NUMSAMP) return "TJPARAM_SUBSAMP is not set";
  if (subsamp != TJSAMP_GRAY && (!dstPlanes[1] || !dstPlanes[2])) return "an argument the reference refuses";
  if (pixelFormat == TJPF_CMYK) return "CMYK pixels";
  if (get(handle, TJPARAM_BOTTOMUP) == 1) return "bottom-up rows";
  if (get(handle, TJPARAM_LOSSLESS) == 1) return "lossless mode";
  /* setCompDefaults: pf2cs, jpeg_set_defaults under JCP_FASTEST, the colour space, the luma sampling factors */
  static const int pf2cs[TJ_NUMPF] = { B200JPEG_CS_EXT_RGB, B200JPEG_CS_EXT_BGR, B200JPEG_CS_EXT_RGBX, B200JPEG_CS_EXT_BGRX,
    B200JPEG_CS_EXT_XBGR, B200JPEG_CS_EXT_XRGB, B200JPEG_CS_GRAYSCALE, B200JPEG_CS_EXT_RGBA, B200JPEG_CS_EXT_BGRA,
    B200JPEG_CS_EXT_ABGR, B200JPEG_CS_EXT_ARGB, B200JPEG_CS_CMYK };
  static const int tjcs2cs[TJ_NUMCS] = { B200JPEG_CS_RGB, B200JPEG_CS_YCbCr, B200JPEG_CS_GRAYSCALE, B200JPEG_CS_CMYK, B200JPEG_CS_YCCK };
  b200jpeg_params p;
  memset(&p, 0, sizeof p);
  p.in_color_space = pf2cs[pixelFormat]; p.input_components = tjPixelSize[pixelFormat];
  p.data_precision = 8;
  b200jpeg_set_defaults(&p, B200JPEG_PROFILE_FASTEST);
  p.image_width = width; p.image_height = height;
  const int tjcs = get(handle, TJPARAM_COLORSPACE);
  const int jcs = tjcs >= 0 && tjcs < TJ_NUMCS ? tjcs2cs[tjcs] : subsamp == TJSAMP_GRAY ? B200JPEG_CS_GRAYSCALE : B200JPEG_CS_YCbCr;
  if (b200jpeg_set_colorspace(&p, jcs) != B200JPEG_OK) return b200jpeg_last_error();
  /* the reference writes three planes unless TJSAMP_GRAY: other component counts are its business */
  if (p.num_components != (subsamp == TJSAMP_GRAY ? 1 : 3)) return "component count differs from the subsampling's planes";
  p.comp_info[0].h_samp_factor = tjMCUWidth[subsamp] / 8; p.comp_info[0].v_samp_factor = tjMCUHeight[subsamp] / 8;
  for (int ci = 1; ci < p.num_components; ci++) p.comp_info[ci].h_samp_factor = p.comp_info[ci].v_samp_factor = 1;
  if (b200jpeg_validate(&p) != B200JPEG_OK) return b200jpeg_last_error();
  size_t pitch_b[3] = {0, 0, 0}, stride_b[3] = {0, 0, 0};
  for (int ci = 0; ci < p.num_components; ci++) {
    int pw, ph;
    if (b200jpeg_yuv_plane_dims(&p, ci, &pw, &ph) != B200JPEG_OK) return b200jpeg_last_error();
    const int s = strides && strides[ci] != 0 ? strides[ci] : pw;                 /* turbojpeg.c:1585 */
    if (s < pw) return "plane stride below the plane width";
    pitch_b[ci] = (size_t)s;
  }
  b200jpeg_encoder *enc = take_encoder();
  if (!enc) return b200jpeg_last_error();
  const size_t row_pitch = pitch ? (size_t)pitch : (size_t)width * tjPixelSize[pixelFormat];
  const int rc = b200jpeg_encode_yuv_batch(enc, &p, srcBuf, 0, row_pitch, 0, (uint8_t *const *)dstPlanes, 0, pitch_b, stride_b, 1);
  give_encoder(enc);
  if (rc != B200JPEG_OK) return b200jpeg_last_error();
  if (verbose()) fprintf(stderr, "b200 shim: device path (YUV planes %dx%d, TJSAMP %d, TJPF %d)\n", width, height, subsamp, pixelFormat);
  return NULL;
}

DLLEXPORT int tj3EncodeYUVPlanes8(tjhandle handle, const unsigned char *srcBuf, int width, int pitch, int height,
                                  int pixelFormat, unsigned char **dstPlanes, int *strides)
{
  static tjyuvplanes_fn real;
  if (!real) real = (tjyuvplanes_fn)next_sym("tj3EncodeYUVPlanes8");
  const char *why = encode_yuv_device(handle, srcBuf, width, pitch, height, pixelFormat, dstPlanes, strides);
  if (!why) return 0;
  if (verbose()) fprintf(stderr, "b200 shim: reference path (YUV planes: %s)\n", why);
  if (required()) { fprintf(stderr, "b200 shim: B200_SHIM_REQUIRE=1 and the device path was not taken: %s\n", why); return -1; }
  return real(handle, srcBuf, width, pitch, height, pixelFormat, dstPlanes, strides);
}

/* tj3EncodeYUV8: the planes back to back, rows padded to `align` (turbojpeg.c:1657-1686), then the planes function */
DLLEXPORT int tj3EncodeYUV8(tjhandle handle, const unsigned char *srcBuf, int width, int pitch, int height,
                            int pixelFormat, unsigned char *dstBuf, int align)
{
  static tjyuv8_fn real; static tjget_fn get; static tjplanedim_fn plane_w, plane_h;
  if (!real) real = (tjyuv8_fn)next_sym("tj3EncodeYUV8");
  if (!get) get = (tjget_fn)next_sym("tj3Get");
  if (!plane_w) plane_w = (tjplanedim_fn)next_sym("tj3YUVPlaneWidth");
  if (!plane_h) plane_h = (tjplanedim_fn)next_sym("tj3YUVPlaneHeight");
  const int subsamp = handle ? get(handle, TJPARAM_SUBSAMP) : -1;
  if (!handle || width <= 0 || height <= 0 || !dstBuf || align < 1 || (align & (align - 1)) || subsamp < 0 || subsamp >= TJ_NUMSAMP)
    return real(handle, srcBuf, width, pitch, height, pixelFormat, dstBuf, align);    /* the reference's refusals */
  unsigned char *planes[3] = {dstBuf, NULL, NULL};
  int strides[3] = {0, 0, 0};
  const int pw0 = plane_w(0, width, subsamp), ph0 = plane_h(0, height, subsamp);
  strides[0] = (pw0 + align - 1) & ~(align - 1);
  if (subsamp != TJSAMP_GRAY) {
    const int pw1 = plane_w(1, width, subsamp), ph1 = plane_h(1, height, subsamp);
    strides[1] = strides[2] = (pw1 + align - 1) & ~(align - 1);
    if ((unsigned long long)strides[0] * ph0 > (unsigned long long)INT_MAX || (unsigned long long)strides[1] * ph1 > (unsigned long long)INT_MAX)
      return real(handle, srcBuf, width, pitch, height, pixelFormat, dstBuf, align);
    planes[1] = planes[0] + (size_t)strides[0] * ph0;
    planes[2] = planes[1] + (size_t)strides[1] * ph1;
  }
  return tj3EncodeYUVPlanes8(handle, srcBuf, width, pitch, height, pixelFormat, planes, strides);
}
#endif
