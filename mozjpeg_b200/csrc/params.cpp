// params.cpp -- host-side parameter logic of libb200jpeg (no device code).
//
// The output bytes of the encoder depend on decisions the reference takes in
// jcparam.c / jcext.c / jcmaster.c before any pixel is touched: quantization
// tables from the quality rating, sampling factors per colour space, the
// default progressive script, which passes run.  These functions mirror that
// API (same names minus the prefix, same argument meaning) on a plain struct.
#include "b200jpeg.h"
#include "internal.h"
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <algorithm>

#include "std_tables.inc"

namespace b200 {
thread_local char g_last_error[512] = "";
void set_error(const char *fmt, ...) {
  va_list ap; va_start(ap, fmt); vsnprintf(g_last_error, sizeof g_last_error, fmt, ap); va_end(ap);
}
}  // namespace b200

extern "C" {

const char *b200jpeg_last_error(void) { return b200::g_last_error; }
const char *b200jpeg_version(void) { return "b200jpeg 0.1 (sm_90a)"; }

const unsigned int *b200jpeg_std_quant_tbl(int set_idx, int chroma) {
  static unsigned int tmp[9][2][64];
  static bool init = false;
  if (!init) { for (int s = 0; s < 9; s++) for (int c = 0; c < 2; c++) for (int i = 0; i < 64; i++) tmp[s][c][i] = kBaseQuant[(s * 2 + c) * 64 + i]; init = true; }
  if (set_idx < 0 || set_idx > 8) return nullptr;
  return tmp[set_idx][chroma ? 1 : 0];
}

// jpeg_float_quality_scaling (jcparam.c:334-357)
float b200jpeg_float_quality_scaling(float quality) {
  if (quality <= 0.f) quality = 1.f;
  if (quality > 100.f) quality = 100.f;
  if (quality < 50.f) quality = 5000.f / quality;
  else quality = 200.f - quality * 2.f;
  return quality;
}
// jpeg_quality_scaling (jcparam.c:328-332): float result truncated to int
int b200jpeg_quality_scaling(int quality) { return (int)b200jpeg_float_quality_scaling((float)quality); }

// jpeg_add_quant_table (jcparam.c:31-68)
int b200jpeg_add_quant_table(b200jpeg_params *p, int which_tbl, const unsigned int *basic_table,
                             int scale_factor, int force_baseline) {
  if (which_tbl < 0 || which_tbl >= B200JPEG_NUM_QUANT_TBLS) { b200::set_error("bogus DQT index %d", which_tbl); return B200JPEG_ERR_PARAM; }
  for (int i = 0; i < 64; i++) {
    long temp = ((long)basic_table[i] * scale_factor + 50L) / 100L;
    if (temp <= 0L) temp = 1L;
    if (temp > 32767L) temp = 32767L;
    if (force_baseline && temp > 255L) temp = 255L;
    p->quant_tbl[which_tbl][i] = (uint16_t)temp;
  }
  p->quant_tbl_present[which_tbl] = 1;
  return B200JPEG_OK;
}
// jpeg_set_linear_quality (jcparam.c:311-325): both slots from the master table set
void b200jpeg_set_linear_quality(b200jpeg_params *p, int scale_factor, int force_baseline) {
  b200jpeg_add_quant_table(p, 0, b200jpeg_std_quant_tbl(p->quant_tbl_master_idx, 0), scale_factor, force_baseline);
  b200jpeg_add_quant_table(p, 1, b200jpeg_std_quant_tbl(p->quant_tbl_master_idx, 1), scale_factor, force_baseline);
}
// jpeg_set_quality (jcparam.c:361-373)
void b200jpeg_set_quality(b200jpeg_params *p, int quality, int force_baseline) {
  b200jpeg_set_linear_quality(p, b200jpeg_quality_scaling(quality), force_baseline);
}
// cjpeg's jpeg_default_qtables (rdswitch.c:509-521)
void b200jpeg_default_qtables(b200jpeg_params *p, int force_baseline) {
  b200jpeg_add_quant_table(p, 0, b200jpeg_std_quant_tbl(p->quant_tbl_master_idx, 0), p->q_scale_factor[0], force_baseline);
  b200jpeg_add_quant_table(p, 1, b200jpeg_std_quant_tbl(p->quant_tbl_master_idx, 1), p->q_scale_factor[1], force_baseline);
}

static void set_huff(b200jpeg_huff_tbl *t, const unsigned char *bits, const unsigned char *val) {
  memset(t, 0, sizeof *t);
  memcpy(t->bits, bits, 17);
  int n = 0; for (int l = 1; l <= 16; l++) n += bits[l];
  memcpy(t->huffval, val, n);
  t->present = 1;
}
// std_huff_tables (jstdhuff.c:52-143)
void b200jpeg_std_huff_tables(b200jpeg_params *p) {
  set_huff(&p->dc_huff_tbl[0], kStdHuff_bits_dc_luminance, kStdHuff_val_dc_luminance);
  set_huff(&p->ac_huff_tbl[0], kStdHuff_bits_ac_luminance, kStdHuff_val_ac_luminance);
  set_huff(&p->dc_huff_tbl[1], kStdHuff_bits_dc_chrominance, kStdHuff_val_dc_chrominance);
  set_huff(&p->ac_huff_tbl[1], kStdHuff_bits_ac_chrominance, kStdHuff_val_ac_chrominance);
}

static void set_comp(b200jpeg_params *p, int i, int id, int h, int v, int q, int dc, int ac) {
  b200jpeg_component_info *c = &p->comp_info[i];
  c->component_id = id; c->h_samp_factor = h; c->v_samp_factor = v; c->quant_tbl_no = q; c->dc_tbl_no = dc; c->ac_tbl_no = ac;
}
// jpeg_set_colorspace (jcparam.c:573-652), the colour spaces on the device path
int b200jpeg_set_colorspace(b200jpeg_params *p, int colorspace) {
  p->jpeg_color_space = colorspace;
  p->write_JFIF_header = 0; p->write_Adobe_marker = 0;
  switch (colorspace) {
  case B200JPEG_CS_GRAYSCALE: p->write_JFIF_header = 1; p->num_components = 1; set_comp(p, 0, 1, 1, 1, 0, 0, 0); break;
  case B200JPEG_CS_RGB:
    p->write_Adobe_marker = 1; p->num_components = 3;
    set_comp(p, 0, 0x52, 1, 1, 0, 0, 0); set_comp(p, 1, 0x47, 1, 1, 0, 0, 0); set_comp(p, 2, 0x42, 1, 1, 0, 0, 0); break;
  case B200JPEG_CS_YCbCr:
    p->write_JFIF_header = 1; p->num_components = 3;
    set_comp(p, 0, 1, 2, 2, 0, 0, 0); set_comp(p, 1, 2, 1, 1, 1, 1, 1); set_comp(p, 2, 3, 1, 1, 1, 1, 1); break;
  case B200JPEG_CS_CMYK:
    p->write_Adobe_marker = 1; p->num_components = 4;
    set_comp(p, 0, 0x43, 1, 1, 0, 0, 0); set_comp(p, 1, 0x4D, 1, 1, 0, 0, 0); set_comp(p, 2, 0x59, 1, 1, 0, 0, 0); set_comp(p, 3, 0x4B, 1, 1, 0, 0, 0); break;
  case B200JPEG_CS_YCCK:
    p->write_Adobe_marker = 1; p->num_components = 4;
    set_comp(p, 0, 1, 2, 2, 0, 0, 0); set_comp(p, 1, 2, 1, 1, 1, 1, 1); set_comp(p, 2, 3, 1, 1, 1, 1, 1); set_comp(p, 3, 4, 2, 2, 0, 0, 0); break;
  case B200JPEG_CS_UNKNOWN:
    p->num_components = p->input_components;
    // MAX_COMPONENTS is 10 in the reference (JERR_COMPONENT_COUNT); the parameter block has room for 4
    if (p->num_components < 1 || p->num_components > 10) { b200::set_error("Too many color components: %d, max 10", p->num_components); return B200JPEG_ERR_PARAM; }
    if (p->num_components > B200JPEG_MAX_COMPONENTS) { b200::set_error("%d components: the device path takes at most %d", p->num_components, B200JPEG_MAX_COMPONENTS); return B200JPEG_ERR_UNSUPPORTED; }
    for (int ci = 0; ci < p->num_components; ci++) set_comp(p, ci, ci, 1, 1, 0, 0, 0);
    break;
  default: b200::set_error("unsupported JPEG colorspace %d", colorspace); return B200JPEG_ERR_UNSUPPORTED;
  }
  return B200JPEG_OK;
}
// jpeg_default_colorspace (jcparam.c:526-566)
int b200jpeg_default_colorspace(b200jpeg_params *p) {
  switch (p->in_color_space) {
  case B200JPEG_CS_GRAYSCALE: return b200jpeg_set_colorspace(p, B200JPEG_CS_GRAYSCALE);
  case B200JPEG_CS_RGB:       return b200jpeg_set_colorspace(p, b200::is_lossless(p) ? B200JPEG_CS_RGB : B200JPEG_CS_YCbCr);   // jcparam.c:544-549
  case B200JPEG_CS_YCbCr:     return b200jpeg_set_colorspace(p, B200JPEG_CS_YCbCr);
  case B200JPEG_CS_CMYK:      return b200jpeg_set_colorspace(p, B200JPEG_CS_CMYK);        // by default, no translation
  case B200JPEG_CS_YCCK:      return b200jpeg_set_colorspace(p, B200JPEG_CS_YCCK);
  case B200JPEG_CS_UNKNOWN:   return b200jpeg_set_colorspace(p, B200JPEG_CS_UNKNOWN);
  default:
    if (B200JPEG_CS_IS_RGB(p->in_color_space)) return b200jpeg_set_colorspace(p, b200::is_lossless(p) ? B200JPEG_CS_RGB : B200JPEG_CS_YCbCr);     // jcparam.c:535-549
    b200::set_error("unsupported input colorspace %d", p->in_color_space); return B200JPEG_ERR_UNSUPPORTED;
  }
}

static b200jpeg_scan_info *fill_a_scan(b200jpeg_scan_info *s, int ci, int Ss, int Se, int Ah, int Al) {
  s->comps_in_scan = 1; s->component_index[0] = ci; s->Ss = Ss; s->Se = Se; s->Ah = Ah; s->Al = Al; return s + 1;
}
static b200jpeg_scan_info *fill_scans(b200jpeg_scan_info *s, int n, int Ss, int Se, int Ah, int Al) {
  for (int ci = 0; ci < n; ci++) s = fill_a_scan(s, ci, Ss, Se, Ah, Al);
  return s;
}
static b200jpeg_scan_info *fill_dc_scans(b200jpeg_scan_info *s, int n, int Ah, int Al) {
  if (n <= 4) { s->comps_in_scan = n; for (int ci = 0; ci < n; ci++) s->component_index[ci] = ci; s->Ss = s->Se = 0; s->Ah = Ah; s->Al = Al; return s + 1; }
  return fill_scans(s, n, 0, 0, Ah, Al);
}
// jpeg_search_progression (jcparam.c:733-852): the candidate list the scan
// search (jcmaster.c:773-962) chooses from; jpeg_simple_progression installs it
// when optimize_scans is set.
static bool search_progression(b200jpeg_params *p) {
  int n = p->num_components;
  static const int frequency_split[5] = {2, 8, 5, 12, 18};
  if (!((n == 3 && p->jpeg_color_space == B200JPEG_CS_YCbCr) || n == 1)) return false;
  b200jpeg_scan_info *s = p->scan_info;
  memset(p->scan_info, 0, sizeof p->scan_info);
  const int Al_max_luma = 3, nsplit = 5;
  s = (p->dc_scan_opt_mode == 0) ? fill_dc_scans(s, n, 0, 0) : fill_dc_scans(s, 1, 0, 0);
  s = fill_a_scan(s, 0, 1, 8, 0, 0); s = fill_a_scan(s, 0, 9, 63, 0, 0);
  for (int Al = 0; Al < Al_max_luma; Al++) { s = fill_a_scan(s, 0, 1, 63, Al + 1, Al); s = fill_a_scan(s, 0, 1, 8, 0, Al + 1); s = fill_a_scan(s, 0, 9, 63, 0, Al + 1); }
  s = fill_a_scan(s, 0, 1, 63, 0, 0);
  for (int i = 0; i < nsplit; i++) { s = fill_a_scan(s, 0, 1, frequency_split[i], 0, 0); s = fill_a_scan(s, 0, frequency_split[i] + 1, 63, 0, 0); }
  if (n != 1) {
    const int Al_max_chroma = 2;
    s->comps_in_scan = 2; s->component_index[0] = 1; s->component_index[1] = 2; s->Ss = s->Se = 0; s->Ah = s->Al = 0; s++;
    s = fill_a_scan(s, 1, 0, 0, 0, 0); s = fill_a_scan(s, 2, 0, 0, 0, 0);
    s = fill_a_scan(s, 1, 1, 8, 0, 0); s = fill_a_scan(s, 1, 9, 63, 0, 0); s = fill_a_scan(s, 2, 1, 8, 0, 0); s = fill_a_scan(s, 2, 9, 63, 0, 0);
    for (int Al = 0; Al < Al_max_chroma; Al++) {
      s = fill_a_scan(s, 1, 1, 63, Al + 1, Al); s = fill_a_scan(s, 2, 1, 63, Al + 1, Al);
      s = fill_a_scan(s, 1, 1, 8, 0, Al + 1); s = fill_a_scan(s, 1, 9, 63, 0, Al + 1);
      s = fill_a_scan(s, 2, 1, 8, 0, Al + 1); s = fill_a_scan(s, 2, 9, 63, 0, Al + 1);
    }
    s = fill_a_scan(s, 1, 1, 63, 0, 0); s = fill_a_scan(s, 2, 1, 63, 0, 0);
    for (int i = 0; i < nsplit; i++) {
      s = fill_a_scan(s, 1, 1, frequency_split[i], 0, 0); s = fill_a_scan(s, 1, frequency_split[i] + 1, 63, 0, 0);
      s = fill_a_scan(s, 2, 1, frequency_split[i], 0, 0); s = fill_a_scan(s, 2, frequency_split[i] + 1, 63, 0, 0);
    }
  }
  p->num_scans = (int)(s - p->scan_info);
  return true;
}

int b200jpeg_simple_progression(b200jpeg_params *p) {
  if (p->optimize_scans) {
    if (search_progression(p)) return B200JPEG_OK;
    p->optimize_scans = 0;   // jcparam.c:754 num_scans_luma=0 -> jcapistd.c:53-56 turns the search off
  }
  if (b200::is_lossless(p)) {   // jcparam.c:875-880: lossless off again, colour space re-derived
    p->num_scans = 0;
    b200jpeg_default_colorspace(p);
  }
  int n = p->num_components;
  bool maxc = p->compress_profile == B200JPEG_PROFILE_MAX_COMPRESSION;
  b200jpeg_scan_info *s = p->scan_info;
  memset(p->scan_info, 0, sizeof p->scan_info);
  if (n == 3 && p->jpeg_color_space == B200JPEG_CS_YCbCr) {
    if (maxc) {
      if (p->dc_scan_opt_mode == 0) s = fill_dc_scans(s, n, 0, 0);
      else if (p->dc_scan_opt_mode == 1) { s = fill_a_scan(s, 0, 0, 0, 0, 0); s = fill_a_scan(s, 1, 0, 0, 0, 0); s = fill_a_scan(s, 2, 0, 0, 0, 0); }
      else { s = fill_dc_scans(s, 1, 0, 0); s->comps_in_scan = 2; s->component_index[0] = 1; s->component_index[1] = 2; s->Ss = s->Se = 0; s->Ah = s->Al = 0; s++; }
      s = fill_a_scan(s, 0, 1, 8, 0, 2); s = fill_a_scan(s, 1, 1, 8, 0, 0); s = fill_a_scan(s, 2, 1, 8, 0, 0);
      s = fill_a_scan(s, 0, 9, 63, 0, 2);
      s = fill_a_scan(s, 0, 1, 63, 2, 1); s = fill_a_scan(s, 0, 1, 63, 1, 0);
      s = fill_a_scan(s, 1, 9, 63, 0, 0); s = fill_a_scan(s, 2, 9, 63, 0, 0);
    } else {
      s = fill_dc_scans(s, n, 0, 1);
      s = fill_a_scan(s, 0, 1, 5, 0, 2); s = fill_a_scan(s, 2, 1, 63, 0, 1); s = fill_a_scan(s, 1, 1, 63, 0, 1);
      s = fill_a_scan(s, 0, 6, 63, 0, 2); s = fill_a_scan(s, 0, 1, 63, 2, 1);
      s = fill_dc_scans(s, n, 1, 0);
      s = fill_a_scan(s, 2, 1, 63, 1, 0); s = fill_a_scan(s, 1, 1, 63, 1, 0); s = fill_a_scan(s, 0, 1, 63, 1, 0);
    }
  } else {
    if (maxc) {
      s = fill_dc_scans(s, n, 0, 0);
      s = fill_scans(s, n, 1, 8, 0, 2); s = fill_scans(s, n, 9, 63, 0, 2);
      s = fill_scans(s, n, 1, 63, 2, 1); s = fill_scans(s, n, 1, 63, 1, 0);
    } else {
      s = fill_dc_scans(s, n, 0, 1);
      s = fill_scans(s, n, 1, 5, 0, 2); s = fill_scans(s, n, 6, 63, 0, 2);
      s = fill_scans(s, n, 1, 63, 2, 1);
      s = fill_dc_scans(s, n, 1, 0); s = fill_scans(s, n, 1, 63, 1, 0);
    }
  }
  p->num_scans = (int)(s - p->scan_info);
  return B200JPEG_OK;
}

}  // extern "C"

namespace b200 {
bool is_lossless(const b200jpeg_params *p)
{
  return !p->optimize_scans && p->num_scans > 0 && p->scan_info[0].Ss != 0 && p->scan_info[0].Se == 0;
}

// the script b200jpeg_enable_lossless installs in place of the reference's scan_info == NULL: one scan, marked by the
// unused entry after it (comps_in_scan = -1), which no script the reference can express has
static bool enable_lossless_script(const b200jpeg_params *p)
{
  return p->num_scans == 1 && p->scan_info[1].comps_in_scan == -1;
}

void lossless_start(const b200jpeg_params *in, b200jpeg_params *out)
{
  *out = *in;
  out->smoothing_factor = 0;                                             // jcmaster.c:1077
  b200jpeg_default_colorspace(out);                                      // :1078
  for (int ci = 0; ci < out->num_components && ci < B200JPEG_MAX_COMPONENTS; ci++)
    out->comp_info[ci].h_samp_factor = out->comp_info[ci].v_samp_factor = 1;   // :1079-1081
  out->optimize_coding = 1;                                              // :1091-1094
  // the reference keeps scan_info == NULL after jpeg_enable_lossless and codes one scan of all components as they are
  // AFTER jpeg_default_colorspace (select_scan_parameters, jcmaster.c:500-513); the script stands in for that
  if (enable_lossless_script(in) && out->num_components <= B200JPEG_MAX_COMPONENTS) {
    b200jpeg_scan_info &s = out->scan_info[0];
    s.comps_in_scan = out->num_components;
    for (int k = 0; k < B200JPEG_MAX_COMPONENTS; k++) s.component_index[k] = k < out->num_components ? k : 0;
  }
}
}  // namespace b200

extern "C" {

// jpeg_enable_lossless (jcparam.c:1015-1039)
int b200jpeg_enable_lossless(b200jpeg_params *p, int psv, int pt)
{
  if (psv < 1 || psv > 7 || pt < 0 || pt >= p->data_precision) { b200::set_error("Invalid progression parameters Ss=%d Se=0 Ah=0 Al=%d", psv, pt); return B200JPEG_ERR_PARAM; }
  if (p->num_scans > 0 && !b200::enable_lossless_script(p)) {
    // the reference keeps an installed script next to its lossless flag.  The scan search's script skips
    // validate_script (jcmaster.c:285-291), so the flag stays on beside progressive mode: with the trellis the passes fail
    // ("Bogus buffer control mode"), without it the file gets SOF2 headers over the lossless compressor's data, which
    // the device path does not represent.  Any other script decides by its first entry (jcmaster.c:302-330), which
    // clears the flag for a sequential or progressive script: then the call changes nothing.
    if (p->optimize_scans) {
      if (p->trellis_quant) { b200::set_error("lossless mode needs trellis quantization off (cjpeg -notrellis), as in the reference"); return B200JPEG_ERR_PARAM; }
      b200::set_error("lossless mode beside the scan search's script (the reference writes SOF2 headers over lossless data) is not on the device path");
      return B200JPEG_ERR_UNSUPPORTED;
    }
    return B200JPEG_OK;
  }
  const int n = p->num_components;
  if (n < 1 || n > B200JPEG_MAX_COMPONENTS) { b200::set_error("Too many color components: %d, max 4", n); return B200JPEG_ERR_PARAM; }
  memset(p->scan_info, 0, sizeof p->scan_info);
  b200jpeg_scan_info &s = p->scan_info[0];
  s.comps_in_scan = n;
  for (int k = 0; k < n; k++) s.component_index[k] = k;
  s.Ss = psv; s.Se = 0; s.Ah = 0; s.Al = pt;
  p->scan_info[1].comps_in_scan = -1;
  p->num_scans = 1;
  p->optimize_scans = 0;        // scan_info == NULL turns the scan search off at jpeg_start_compress (jcapistd.c:53-56)
  return B200JPEG_OK;
}

// jpeg_CreateCompress (profile, jcapimin.c:107-109) + jpeg_set_defaults (jcparam.c:386-519)
void b200jpeg_set_defaults(b200jpeg_params *p, int profile) {
  int in_cs = p->in_color_space, in_comp = p->input_components, w = p->image_width, h = p->image_height;
  int prec = p->data_precision ? p->data_precision : 8;
  memset(p, 0, sizeof *p);
  p->in_color_space = in_cs; p->input_components = in_comp; p->image_width = w; p->image_height = h;
  p->data_precision = prec;
  p->compress_profile = profile;
  bool maxc = profile == B200JPEG_PROFILE_MAX_COMPRESSION;
  // Quirk kept from the reference (jcparam.c:411 vs :509): the default q75
  // tables are built BEFORE quant_tbl_master_idx is switched to 3, i.e. from
  // table set 0 (Annex K).  A later set_quality call uses set 3.
  p->quant_tbl_master_idx = 0;
  b200jpeg_set_quality(p, 75, 1);
  b200jpeg_std_huff_tables(p);
  p->num_scans = 0;
  p->optimize_coding = maxc ? 1 : 0;
  if (p->data_precision == 12) p->optimize_coding = 1;
  p->overshoot_deringing = maxc ? 1 : 0;
  p->smoothing_factor = 0;
  p->dct_method = B200JPEG_DCT_ISLOW;          // JDCT_DEFAULT
  p->restart_interval = 0; p->restart_in_rows = 0;
  p->JFIF_major_version = 1; p->JFIF_minor_version = 1;
  p->density_unit = 0; p->X_density = 1; p->Y_density = 1;
  b200jpeg_default_colorspace(p);
  p->dc_scan_opt_mode = 0;
  p->optimize_scans = maxc ? 1 : 0;
  if (maxc) b200jpeg_simple_progression(p);     // jcparam.c:496-500 (installs the search script)
  p->trellis_quant = maxc ? 1 : 0;
  p->lambda_log_scale1 = 14.75f; p->lambda_log_scale2 = 16.5f;
  p->quant_tbl_master_idx = maxc ? 3 : 0;
  p->use_lambda_weight_tbl = 1; p->use_scans_in_trellis = 0;
  p->trellis_freq_split = 8; p->trellis_num_loops = 1;
  p->trellis_q_opt = 0; p->trellis_quant_dc = 1; p->trellis_delta_dc_weight = 0.0f;
  for (int i = 0; i < 4; i++) p->q_scale_factor[i] = 100;
}

static int div_round_up(long a, long b) { return (int)((a + b - 1) / b); }

// validate_script's lossless branch (jcmaster.c:302-311, :389-415) on the script as given, before the start-time overrides
static int validate_lossless_script(const b200jpeg_params *p)
{
  using b200::set_error;
  if (p->num_scans > B200JPEG_MAX_SCANS) { set_error("Invalid scan script at entry 0"); return B200JPEG_ERR_PARAM; }
  bool sent[4] = {false, false, false, false};
  const b200jpeg_scan_info *s = p->scan_info;
  for (int scanno = 1; scanno <= p->num_scans; scanno++, s++) {
    const int n = s->comps_in_scan;
    if (n <= 0 || n > 4) { set_error("Too many color components: %d, max 4", n); return B200JPEG_ERR_PARAM; }
    for (int ci = 0; ci < n; ci++) {
      const int t = s->component_index[ci];
      if (t < 0 || t >= p->num_components || (ci > 0 && t <= s->component_index[ci - 1])) { set_error("Invalid scan script at entry %d", scanno); return B200JPEG_ERR_PARAM; }
    }
    if (s->Ss < 1 || s->Ss > 7 || s->Se != 0 || s->Ah != 0 || s->Al < 0 || s->Al >= p->data_precision) { set_error("Invalid progressive parameters at scan script entry %d", scanno); return B200JPEG_ERR_PARAM; }
    for (int ci = 0; ci < n; ci++) { const int t = s->component_index[ci]; if (sent[t]) { set_error("Invalid scan script at entry %d", scanno); return B200JPEG_ERR_PARAM; } sent[t] = true; }
  }
  for (int ci = 0; ci < p->num_components && ci < 4; ci++) if (!sent[ci]) { set_error("Scan script does not transmit all data"); return B200JPEG_ERR_PARAM; }
  return B200JPEG_OK;
}

static int validate_effective(const b200jpeg_params *p, bool lossless);

int b200jpeg_validate(const b200jpeg_params *p) {
  using b200::set_error;
  const bool lossless = b200::is_lossless(p);
  if (lossless) {
    if (p->num_components > 10) { set_error("Too many color components: %d, max 10", p->num_components); return B200JPEG_ERR_PARAM; }
    if (p->num_components > B200JPEG_MAX_COMPONENTS) { set_error("%d components: the device path takes at most %d", p->num_components, B200JPEG_MAX_COMPONENTS); return B200JPEG_ERR_UNSUPPORTED; }
    if (p->data_precision != 8 && p->data_precision != 12 && p->data_precision != 16) { set_error("Unsupported JPEG data precision %d", p->data_precision); return B200JPEG_ERR_PARAM; }
    int rc = validate_lossless_script(p);
    if (rc) return rc;
    // the rest is checked on the block jpeg_start_compress works with
    b200jpeg_params eff;
    b200::lossless_start(p, &eff);
    return validate_effective(&eff, true);
  }
  return validate_effective(p, false);
}

// everything validate checks on the parameter block jpeg_start_compress works with
static int validate_effective(const b200jpeg_params *p, const bool lossless) {
  using b200::set_error;
  if (lossless) {
    if (p->num_components > B200JPEG_MAX_COMPONENTS) { set_error("%d components: the device path takes at most %d", p->num_components, B200JPEG_MAX_COMPONENTS); return B200JPEG_ERR_UNSUPPORTED; }
    // the difference controller has no JBUF_REQUANT mode (jcdiffct.c:116-137): the trellis passes fail with "Bogus buffer control mode"
    if (p->trellis_quant) { set_error("lossless mode needs trellis quantization off (cjpeg -notrellis), as in the reference"); return B200JPEG_ERR_PARAM; }
  }
  // initial_setup (jcmaster.c:169-249)
  if (p->image_height <= 0 || p->image_width <= 0 || p->num_components <= 0 || p->input_components <= 0) { set_error("Empty input image"); return B200JPEG_ERR_PARAM; }
  if (p->image_height > 65500 || p->image_width > 65500) { set_error("Maximum supported image dimension is 65500 pixels"); return B200JPEG_ERR_PARAM; }
  // 16-bit samples exist in lossless mode only (jcinit.c:95-96)
  if (p->data_precision != 8 && p->data_precision != 12 && !(lossless && p->data_precision == 16)) { set_error("Unsupported JPEG data precision %d", p->data_precision); return B200JPEG_ERR_PARAM; }   // JERR_BAD_PRECISION
  // 12-bit: the coefficient controller has no JBUF_REQUANT mode (jccoefct.c:132-138), so the reference cannot run the
  // trellis passes ("Bogus buffer control mode"); its 12-bit deringing is unusable (jcdctmgr.c:419)
  if (!lossless && p->data_precision == 12 && (p->trellis_quant || p->overshoot_deringing)) { set_error("12-bit precision needs trellis quantization and overshoot deringing off (cjpeg -notrellis -noovershoot), as in the reference"); return B200JPEG_ERR_PARAM; }
  if (p->num_components > 10) { set_error("Too many color components: %d, max 10", p->num_components); return B200JPEG_ERR_PARAM; }   // JERR_COMPONENT_COUNT
  if (p->num_components > B200JPEG_MAX_COMPONENTS) { set_error("%d components: the device path takes at most %d", p->num_components, B200JPEG_MAX_COMPONENTS); return B200JPEG_ERR_UNSUPPORTED; }
  int hmax = 1, vmax = 1;
  for (int ci = 0; ci < p->num_components; ci++) {
    const b200jpeg_component_info *c = &p->comp_info[ci];
    if (c->h_samp_factor <= 0 || c->h_samp_factor > 4 || c->v_samp_factor <= 0 || c->v_samp_factor > 4) { set_error("Bogus sampling factors"); return B200JPEG_ERR_PARAM; }
    if (c->h_samp_factor > hmax) hmax = c->h_samp_factor;
    if (c->v_samp_factor > vmax) vmax = c->v_samp_factor;
    if (!lossless && (c->quant_tbl_no < 0 || c->quant_tbl_no >= 4 || !p->quant_tbl_present[c->quant_tbl_no])) { set_error("Quantization table 0x%02x was not defined", c->quant_tbl_no); return B200JPEG_ERR_PARAM; }
    if (c->dc_tbl_no < 0 || c->dc_tbl_no >= 4 || c->ac_tbl_no < 0 || c->ac_tbl_no >= 4) { set_error("Huffman table index out of range"); return B200JPEG_ERR_PARAM; }
  }
  int blocks_in_mcu = 0;
  for (int ci = 0; ci < p->num_components; ci++) {
    const b200jpeg_component_info *c = &p->comp_info[ci];
    if (hmax % c->h_samp_factor || vmax % c->v_samp_factor) { set_error("Fractional sampling not implemented yet"); return B200JPEG_ERR_PARAM; }   // jcsample.c:535
    blocks_in_mcu += c->h_samp_factor * c->v_samp_factor;
  }
  if (blocks_in_mcu > 10) { set_error("Sampling factors too large for interleaved scan"); return B200JPEG_ERR_PARAM; }   // C_MAX_BLOCKS_IN_MCU
  // jinit_color_converter (jccolor.c:551-740), its two switches: input_components against in_color_space ...
  const int in_cs = p->in_color_space, jcs = p->jpeg_color_space, nc = p->num_components;
  int in_size = 0;                                    // 0: any count (JCS_UNKNOWN and values the reference does not name)
  if (B200JPEG_CS_IS_RGB(in_cs)) in_size = B200JPEG_CS_PIXELSIZE(in_cs);   // rgb_pixelsize[]
  else if (in_cs == B200JPEG_CS_GRAYSCALE) in_size = 1;
  else if (in_cs == B200JPEG_CS_YCbCr) in_size = 3;
  else if (in_cs == B200JPEG_CS_CMYK || in_cs == B200JPEG_CS_YCCK) in_size = 4;
  if (in_size && p->input_components != in_size) { set_error("Bogus input colorspace"); return B200JPEG_ERR_PARAM; }
  // ... then num_components against jpeg_color_space, and the conversions it implements
  bool conv;
  if (lossless) {
    // only the null-type conversions exist in lossless mode (jccolor.c:604-715: JERR_CONVERSION_NOTIMPL otherwise)
    const int want = jcs == B200JPEG_CS_GRAYSCALE ? 1 : jcs == B200JPEG_CS_RGB || jcs == B200JPEG_CS_YCbCr ? 3 : jcs == B200JPEG_CS_CMYK || jcs == B200JPEG_CS_YCCK ? 4 : p->input_components;
    if (nc != want) { set_error("Bogus JPEG colorspace"); return B200JPEG_ERR_PARAM; }
    conv = jcs == B200JPEG_CS_RGB ? B200JPEG_CS_IS_RGB(in_cs) : jcs == in_cs;
    if (!conv) { set_error("Unsupported color conversion request"); return B200JPEG_ERR_PARAM; }
  } else
  switch (jcs) {
  case B200JPEG_CS_GRAYSCALE:
    if (nc != 1) { set_error("Bogus JPEG colorspace"); return B200JPEG_ERR_PARAM; }
    conv = in_cs == B200JPEG_CS_GRAYSCALE || B200JPEG_CS_IS_RGB(in_cs) || in_cs == B200JPEG_CS_YCbCr; break;
  case B200JPEG_CS_RGB:
    if (nc != 3) { set_error("Bogus JPEG colorspace"); return B200JPEG_ERR_PARAM; }
    conv = B200JPEG_CS_IS_RGB(in_cs); break;
  case B200JPEG_CS_YCbCr:
    if (nc != 3) { set_error("Bogus JPEG colorspace"); return B200JPEG_ERR_PARAM; }
    conv = B200JPEG_CS_IS_RGB(in_cs) || in_cs == B200JPEG_CS_YCbCr; break;
  case B200JPEG_CS_CMYK:
    if (nc != 4) { set_error("Bogus JPEG colorspace"); return B200JPEG_ERR_PARAM; }
    conv = in_cs == B200JPEG_CS_CMYK; break;
  case B200JPEG_CS_YCCK:
    if (nc != 4) { set_error("Bogus JPEG colorspace"); return B200JPEG_ERR_PARAM; }
    conv = in_cs == B200JPEG_CS_CMYK || in_cs == B200JPEG_CS_YCCK; break;
  default:                                            // null conversion of JCS_UNKNOWN
    conv = jcs == in_cs && nc == p->input_components;
    if (conv && jcs != B200JPEG_CS_UNKNOWN) { set_error("null conversion of colour space %d: the device path takes it for JCS_UNKNOWN only", jcs); return B200JPEG_ERR_UNSUPPORTED; }
  }
  if (!conv) { set_error("Unsupported color conversion request"); return B200JPEG_ERR_PARAM; }
  // things the reference can do that the device path cannot (yet)
  if (p->restart_interval < 0 || p->restart_interval > 65535 || p->restart_in_rows < 0) { set_error("restart interval out of range"); return B200JPEG_ERR_PARAM; }
  if (lossless) {
    // the restart interval of every scan (jcmaster.c:595-600) must be whole rows: MCUs_per_row is the image width, all
    // components being 1x1 (start_pass_lossless, jclossls.c:292-294: JERR_BAD_RESTART)
    const int ri = p->restart_in_rows > 0 ? (int)std::min((long)p->restart_in_rows * p->image_width, 65535L) : p->restart_interval;
    if (ri % p->image_width) { set_error("Restart interval %d is not a multiple of the number of MCUs per row (%d)", ri, p->image_width); return B200JPEG_ERR_PARAM; }
    return B200JPEG_OK;
  }
  if (p->dct_method < B200JPEG_DCT_ISLOW || p->dct_method > B200JPEG_DCT_FLOAT) { set_error("unknown dct_method %d", p->dct_method); return B200JPEG_ERR_PARAM; }
  if (p->smoothing_factor < 0 || p->smoothing_factor > 100) { set_error("smoothing_factor %d out of range 0..100", p->smoothing_factor); return B200JPEG_ERR_PARAM; }
  if (p->trellis_quant && p->use_scans_in_trellis && (p->trellis_freq_split < 1 || p->trellis_freq_split > 62)) { set_error("trellis_freq_split %d: the device path takes 1..62 with use_scans_in_trellis", p->trellis_freq_split); return B200JPEG_ERR_UNSUPPORTED; }
  if (p->trellis_num_loops < 1 || p->trellis_num_loops > 16) { set_error("trellis_num_loops %d: the device path takes 1..16", p->trellis_num_loops); return B200JPEG_ERR_UNSUPPORTED; }
  // validate_script (jcmaster.c:252-436)
  bool progressive = false;
  if (p->num_scans > 0 && p->optimize_scans) {
    // "When we optimize scans, there is redundancy in the scan list and this function will fail.
    //  Therefore skip all this checking" (jcmaster.c:285-291); the device path wants exactly the search script
    progressive = true;
    if (p->num_scans != (p->num_components == 1 ? 23 : 64) || (p->num_components != 1 && p->num_components != 3)) { set_error("optimize_scans needs the candidate script of jpeg_search_progression (jpeg_simple_progression with optimize_scans set)"); return B200JPEG_ERR_UNSUPPORTED; }
    {
      // the plan indexes components and MCU slots straight from the entries: they must be the search script itself
      static thread_local b200jpeg_params ref;
      ref = *p;
      if (!search_progression(&ref) || ref.num_scans != p->num_scans) { set_error("optimize_scans needs the candidate script of jpeg_search_progression"); return B200JPEG_ERR_UNSUPPORTED; }
      for (int i = 0; i < p->num_scans; i++) {
        const b200jpeg_scan_info &a = p->scan_info[i], &b = ref.scan_info[i];
        bool same = a.comps_in_scan == b.comps_in_scan && a.Ss == b.Ss && a.Se == b.Se && a.Ah == b.Ah && a.Al == b.Al;
        for (int k = 0; same && k < b.comps_in_scan; k++) same = a.component_index[k] == b.component_index[k];
        if (!same) { set_error("optimize_scans: scan script entry %d is not the candidate jpeg_search_progression generates", i + 1); return B200JPEG_ERR_UNSUPPORTED; }
      }
    }
  } else if (p->num_scans > 0) {
    if (p->num_scans > B200JPEG_MAX_SCANS) { set_error("Invalid scan script at entry 0"); return B200JPEG_ERR_PARAM; }
    const b200jpeg_scan_info *s = p->scan_info;
    if (s->Ss != 0 && s->Se == 0) { set_error("lossless scan script is out of scope"); return B200JPEG_ERR_UNSUPPORTED; }
    progressive = (s->Ss != 0 || s->Se != 63);
    int last_bitpos[4][64]; bool sent[4] = {false, false, false, false};
    for (int ci = 0; ci < 4; ci++) for (int k = 0; k < 64; k++) last_bitpos[ci][k] = -1;
    for (int scanno = 1; scanno <= p->num_scans; scanno++, s++) {
      int n = s->comps_in_scan;
      if (n <= 0 || n > 4) { set_error("Too many color components: %d, max 4", n); return B200JPEG_ERR_PARAM; }
      for (int ci = 0; ci < n; ci++) {
        int t = s->component_index[ci];
        if (t < 0 || t >= p->num_components || (ci > 0 && t <= s->component_index[ci - 1])) { set_error("Invalid scan script at entry %d", scanno); return B200JPEG_ERR_PARAM; }
      }
      if (progressive) {
        if (s->Ss < 0 || s->Ss >= 64 || s->Se < s->Ss || s->Se >= 64 || s->Ah < 0 || s->Ah > 10 || s->Al < 0 || s->Al > 10) { set_error("Invalid progressive parameters at scan script entry %d", scanno); return B200JPEG_ERR_PARAM; }
        if (s->Ss == 0) { if (s->Se != 0) { set_error("Invalid progressive parameters at scan script entry %d", scanno); return B200JPEG_ERR_PARAM; } }
        else if (n != 1) { set_error("Invalid progressive parameters at scan script entry %d", scanno); return B200JPEG_ERR_PARAM; }
        for (int ci = 0; ci < n; ci++) {
          int *lb = last_bitpos[s->component_index[ci]];
          if (s->Ss != 0 && lb[0] < 0) { set_error("Invalid progressive parameters at scan script entry %d", scanno); return B200JPEG_ERR_PARAM; }
          for (int k = s->Ss; k <= s->Se; k++) {
            if (lb[k] < 0) { if (s->Ah != 0) { set_error("Invalid progressive parameters at scan script entry %d", scanno); return B200JPEG_ERR_PARAM; } }
            else if (s->Ah != lb[k] || s->Al != s->Ah - 1) { set_error("Invalid progressive parameters at scan script entry %d", scanno); return B200JPEG_ERR_PARAM; }
            lb[k] = s->Al;
          }
        }
      } else {
        if (s->Ss != 0 || s->Se != 63 || s->Ah != 0 || s->Al != 0) { set_error("Invalid progressive parameters at scan script entry %d", scanno); return B200JPEG_ERR_PARAM; }
        for (int ci = 0; ci < n; ci++) { int t = s->component_index[ci]; if (sent[t]) { set_error("Invalid scan script at entry %d", scanno); return B200JPEG_ERR_PARAM; } sent[t] = true; }
      }
    }
    if (progressive) { for (int ci = 0; ci < p->num_components; ci++) if (last_bitpos[ci][0] < 0) { set_error("Scan script does not transmit all data"); return B200JPEG_ERR_PARAM; } }
    else { for (int ci = 0; ci < p->num_components; ci++) if (!sent[ci]) { set_error("Scan script does not transmit all data"); return B200JPEG_ERR_PARAM; } }
  }
  bool optimize = p->optimize_coding || progressive;
  if (p->data_precision == 12) optimize = true;                     // jcmaster.c:1102-1105
  if (p->trellis_quant && !optimize) { set_error("trellis quantization without optimize_coding is not on the device path yet"); return B200JPEG_ERR_UNSUPPORTED; }
  if (!optimize) {
    for (int ci = 0; ci < p->num_components; ci++) {
      const b200jpeg_component_info *c = &p->comp_info[ci];
      if (!p->dc_huff_tbl[c->dc_tbl_no].present || !p->ac_huff_tbl[c->ac_tbl_no].present) { set_error("Huffman table 0x%02x was not defined", c->dc_tbl_no); return B200JPEG_ERR_PARAM; }
    }
  }
  (void)div_round_up;
  return B200JPEG_OK;
}

// jinit_c_master_control pass accounting (jcmaster.c:1114-1139)
int b200jpeg_total_passes(const b200jpeg_params *p) {
  bool progressive = p->num_scans > 0 && (p->scan_info[0].Ss != 0 || p->scan_info[0].Se != 63);
  bool optimize = p->optimize_coding || progressive;
  int num_scans = p->num_scans > 0 ? p->num_scans : 1;
  int total = optimize ? num_scans * 2 : num_scans;
  if (p->trellis_quant) {
    const int per = p->use_scans_in_trellis ? 2 : 1;                      // jcmaster.c:1128-1139
    int base = optimize ? 2 * per * p->num_components * p->trellis_num_loops : per * p->num_components * p->trellis_num_loops + 1;
    total += base;
  }
  return total;
}

}  // extern "C"
