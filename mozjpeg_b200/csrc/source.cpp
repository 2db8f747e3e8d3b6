// source.cpp -- the source side of jpegtran: the marker parser of a JPEG file (jdmarker.c read_markers over the whole
// file) and the host half of the device entropy decode, which cuts every scan into restart segments, removes the
// stuffed zero bytes while copying them into the upload buffer and derives the Huffman decode tables.
#include "b200jpeg.h"
#include "internal.h"
#include <algorithm>
#include <cstring>
#include <map>
#include <string>

namespace b200 {

static const int kNatural[64] = {
   0,  1,  8, 16,  9,  2,  3, 10, 17, 24, 32, 25, 18, 11,  4,  5,
  12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,  6,  7, 14, 21, 28,
  35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
  58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// jpeg_make_d_derived_tbl (jdhuff.c:143-261) with its validation; -1 where it raises JERR_BAD_HUFF_TABLE
int derive_dec_table(const b200jpeg_huff_tbl &h, bool is_dc, DecTable *out)
{
  int huffsize[257], huffcode[257], p = 0;
  for (int l = 1; l <= 16; l++) {
    const int i = h.bits[l];
    if (p + i > 256) return -1;
    for (int k = 0; k < i; k++) huffsize[p++] = l;
  }
  huffsize[p] = 0;
  const int nsym = p;
  unsigned code = 0; int si = huffsize[0]; p = 0;
  while (huffsize[p]) {
    while (huffsize[p] == si) { huffcode[p++] = (int)code; code++; }
    if ((long long)code >= (1LL << si)) return -1;
    code <<= 1; si++;
  }
  if (is_dc) for (int i = 0; i < nsym; i++) if (h.huffval[i] > 15) return -1;
  if (!out) return 0;
  memset(out, 0, sizeof *out);
  p = 0;
  for (int l = 1; l <= 16; l++) {
    if (h.bits[l]) { out->valoff[l] = p - huffcode[p]; p += h.bits[l]; out->maxcode[l] = huffcode[p - 1]; }
    else out->maxcode[l] = -1;
  }
  out->maxcode[17] = 0xFFFFF;
  p = 0;
  for (int l = 1; l <= 8; l++)
    for (int i = 1; i <= h.bits[l]; i++, p++) {
      int look = huffcode[p] << (8 - l);
      for (int c = 1 << (8 - l); c > 0; c--) out->look[look++] = (uint16_t)(l << 8 | h.huffval[p]);
    }
  memcpy(out->huffval, h.huffval, 256);
  return 0;
}

static int bad(int code, const char *msg) { set_error("%s", msg); return code; }
static unsigned be16(const uint8_t *d) { return (unsigned)d[0] << 8 | d[1]; }

// end of the entropy-coded data starting at `pos`: the first 0xFF that starts a marker other than RSTn (a run of fill
// bytes in front of it belongs to the marker).  Fill bytes are allowed only in front of a marker: FF FF 00 is where the
// reference's decoder hits a marker (decode_mcu_fast, jdhuff.c GET_BYTE), so the data ends there too.
static size_t scan_data_end(const uint8_t *d, size_t n, size_t pos)
{
  while (pos < n) {
    const uint8_t *f = static_cast<const uint8_t *>(memchr(d + pos, 0xFF, n - pos));
    if (!f) return n;
    size_t q = (size_t)(f - d), r = q + 1;
    while (r < n && d[r] == 0xFF) r++;
    if (r >= n) return q;
    if ((d[r] == 0x00 && r == q + 1) || (d[r] >= 0xD0 && d[r] <= 0xD7)) { pos = r + 1; continue; }
    return q;
  }
  return n;
}

}  // namespace b200

using namespace b200;

// b200jpeg_parse_source; markers (or nullptr): receives, in file order, the COM and APPn segments (marker, length,
// data) a decompress object with jpeg_save_markers on all of them holds once jpeg_start_decompress returns, which is
// what rdjpeg.c hands cjpeg to copy: those in front of the first SOS and, for a file of several scans, which
// jpeg_start_decompress reads to its end (jdapistd.c:80-103), the later ones too
static int parse_source(const uint8_t *d, size_t n, b200jpeg_source_info *s, std::vector<uint8_t> *markers)
{
  if (!d || !s) return bad(B200JPEG_ERR_PARAM, "bad argument");
  struct Saved { size_t pos, len; int scans_seen; };
  std::vector<Saved> saved;
  memset(s, 0, sizeof *s);
  s->data_precision = 8; s->JFIF_major_version = 1; s->JFIF_minor_version = 1; s->X_density = s->Y_density = 1;
  if (n < 2 || d[0] != 0xFF || d[1] != 0xD8) return bad(B200JPEG_ERR_PARAM, "not a JPEG file");
  int htab[2][4]; for (int c = 0; c < 2; c++) for (int t = 0; t < 4; t++) htab[c][t] = -1;   // [is_ac][slot] -> pool index
  uint16_t qcur[4][64]; int qdef[4] = {0, 0, 0, 0};
  bool saw_sof = false, saw_sos = false;
  int ri = 0;
  size_t pos = 2;
  while (pos + 4 <= n) {
    if (d[pos] != 0xFF) return bad(B200JPEG_ERR_PARAM, "corrupt JPEG header");
    const int m = d[pos + 1];
    if (m == 0xFF) { pos++; continue; }
    if (m == 0x00) return bad(B200JPEG_ERR_BAD_SOURCE, "0xFF 0x00 where a marker is due (fill bytes inside entropy-coded data)");
    if (m == 0xD9) break;                                                      // EOI
    if (m == 0x01 || (m >= 0xD0 && m <= 0xD7)) { pos += 2; continue; }         // TEM, stray RSTn: parameterless (jdmarker.c:1091-1101)
    const size_t ln = be16(d + pos + 2);
    if (ln < 2 || pos + 2 + ln > n) return bad(B200JPEG_ERR_PARAM, "corrupt JPEG header");
    const uint8_t *seg = d + pos + 4; const size_t sl = ln - 2;
    if (m == 0xC0 || m == 0xC1 || m == 0xC2) {
      if (saw_sof || sl < 6) return bad(B200JPEG_ERR_BAD_SOURCE, "bad or repeated SOF marker");
      saw_sof = true; s->sof = m;
      s->data_precision = seg[0]; s->image_height = (int)be16(seg + 1); s->image_width = (int)be16(seg + 3);
      const int nc = seg[5];
      if (nc != 1 && nc != 3 && nc != 4) return bad(B200JPEG_ERR_UNSUPPORTED, "only 1-, 3- and 4-component files are on the device path");
      if (sl < 6 + 3 * (size_t)nc) return bad(B200JPEG_ERR_PARAM, "corrupt JPEG header");
      s->num_components = nc;
      for (int i = 0; i < nc; i++) {
        s->component_id[i] = seg[6 + 3 * i]; s->h_samp_factor[i] = seg[7 + 3 * i] >> 4; s->v_samp_factor[i] = seg[7 + 3 * i] & 15;
        s->quant_tbl_no[i] = seg[8 + 3 * i];
        if (s->h_samp_factor[i] < 1 || s->h_samp_factor[i] > 4 || s->v_samp_factor[i] < 1 || s->v_samp_factor[i] > 4 || s->quant_tbl_no[i] > 3)
          return bad(B200JPEG_ERR_BAD_SOURCE, "bogus sampling factors or quantization table number in SOF");
      }
      if (s->image_height <= 0 || s->image_width <= 0) return bad(B200JPEG_ERR_BAD_SOURCE, "empty image (SOF height or width 0)");   // JERR_EMPTY_IMAGE
      if (s->data_precision != 8 && s->data_precision != 12) return bad(B200JPEG_ERR_BAD_SOURCE, "unsupported JPEG data precision");
    } else if (m == 0xC3 || (m >= 0xC5 && m <= 0xC7) || (m >= 0xC9 && m <= 0xCB) || (m >= 0xCD && m <= 0xCF)) {
      return bad(B200JPEG_ERR_UNSUPPORTED, "lossless / hierarchical / arithmetic-coded source files are out of scope");
    } else if (m == 0xDB) {
      size_t q = 0;
      while (q < sl) {
        const int pq = seg[q] >> 4, tq = seg[q] & 15; q++;
        if (tq > 3 || pq > 1 || q + 64 * (pq + 1) > sl) return bad(B200JPEG_ERR_BAD_SOURCE, "bogus DQT");
        for (int k = 0; k < 64; k++) { qcur[tq][kNatural[k]] = (uint16_t)(pq ? be16(seg + q) : seg[q]); q += pq + 1; }
        qdef[tq] = 1;
        if (!saw_sos) { memcpy(s->quant_tbl[tq], qcur[tq], sizeof qcur[tq]); s->quant_tbl_present[tq] = 1; }
      }
    } else if (m == 0xC4) {
      size_t q = 0;
      while (q < sl) {
        if (q + 17 > sl) return bad(B200JPEG_ERR_BAD_SOURCE, "bogus DHT");
        int idx = seg[q]; const int is_ac = (idx & 0x10) != 0; idx &= ~0x10;
        if (idx < 0 || idx > 3) return bad(B200JPEG_ERR_BAD_SOURCE, "bogus DHT index");   // JERR_DHT_INDEX
        if (s->num_huff >= B200JPEG_MAX_SOURCE_HUFF) return bad(B200JPEG_ERR_UNSUPPORTED, "too many Huffman table definitions");
        b200jpeg_huff_tbl &h = s->huff[s->num_huff];
        int count = 0;
        for (int l = 1; l <= 16; l++) { h.bits[l] = seg[q + l]; count += seg[q + l]; }
        q += 17;
        if (count > 256 || q + count > sl) return bad(B200JPEG_ERR_BAD_SOURCE, "bogus DHT counts");   // JERR_BAD_HUFF_TABLE
        memcpy(h.huffval, seg + q, count); q += count;
        h.present = 1;
        s->huff_is_dc[s->num_huff] = !is_ac;
        htab[is_ac][idx] = s->num_huff++;
      }
    } else if (m == 0xDD) {
      if (sl != 2) return bad(B200JPEG_ERR_BAD_SOURCE, "bogus DRI length");
      ri = (int)be16(seg);
    } else if (m == 0xDC) {
      // DNL: ignored, like the reference (jdmarker.c:1104)
    } else if (m == 0xE0 || m == 0xEE || m == 0xFE || (m >= 0xE1 && m <= 0xEF)) {
      if (markers) saved.push_back({pos, 2 + ln, s->num_scans});
      if (m == 0xE0 && sl >= 14 && !memcmp(seg, "JFIF\0", 5)) {
        s->saw_JFIF = 1; s->JFIF_major_version = seg[5]; s->JFIF_minor_version = seg[6];
        s->density_unit = seg[7]; s->X_density = (int)be16(seg + 8); s->Y_density = (int)be16(seg + 10);
      } else if (m == 0xEE && sl >= 12 && !memcmp(seg, "Adobe", 5)) {
        s->saw_Adobe = 1; s->Adobe_transform = seg[11];
      } else if (m == 0xFE || (m >= 0xE0 && m <= 0xEF)) {
        s->has_extra_markers = 1;
      }
    } else if (m == 0xDA) {
      if (!saw_sof) return bad(B200JPEG_ERR_BAD_SOURCE, "SOS before SOF");
      if (s->num_scans >= B200JPEG_MAX_SOURCE_SCANS) return bad(B200JPEG_ERR_UNSUPPORTED, "too many scans");
      if (!saw_sos && s->sof != 0xC2) {
        // jinit_huff_decoder's std_huff_tables (jdhuff.c:819-823, jstdhuff.c:26-29): the standard tables go into the
        // slots 0 and 1 the file has not defined by its first SOS (Motion-JPEG frames carry no DHT)
        b200jpeg_params sp; memset(&sp, 0, sizeof sp);
        b200jpeg_std_huff_tables(&sp);
        for (int is_ac = 0; is_ac < 2; is_ac++)
          for (int t = 0; t < 2; t++) {
            if (htab[is_ac][t] >= 0) continue;
            if (s->num_huff >= B200JPEG_MAX_SOURCE_HUFF) return bad(B200JPEG_ERR_UNSUPPORTED, "too many Huffman table definitions");
            s->huff[s->num_huff] = is_ac ? sp.ac_huff_tbl[t] : sp.dc_huff_tbl[t];
            s->huff_is_dc[s->num_huff] = !is_ac;
            htab[is_ac][t] = s->num_huff++;
          }
      }
      b200jpeg_source_scan &sc = s->scans[s->num_scans];
      const int ns = sl ? seg[0] : 0;
      if (ns < 1 || ns > 4 || sl != (size_t)(4 + 2 * ns)) return bad(B200JPEG_ERR_BAD_SOURCE, "bogus SOS");
      sc.comps_in_scan = ns;
      for (int i = 0; i < ns; i++) {
        const int cid = seg[1 + 2 * i], td = seg[2 + 2 * i] >> 4, ta = seg[2 + 2 * i] & 15;
        int ci = -1;
        for (int c = 0; c < s->num_components; c++) if (s->component_id[c] == cid) ci = c;
        for (int j = 0; j < i; j++) if (sc.component_index[j] == ci) ci = -1;
        if (ci < 0 || td > 3 || ta > 3) return bad(B200JPEG_ERR_BAD_SOURCE, "SOS names an unknown or repeated component or a bad table number");
        sc.component_index[i] = ci; sc.dc_tbl_no[i] = td; sc.ac_tbl_no[i] = ta;
        sc.dc_huff[i] = htab[0][td]; sc.ac_huff[i] = htab[1][ta];
      }
      sc.Ss = seg[1 + 2 * ns]; sc.Se = seg[2 + 2 * ns]; sc.Ah = seg[3 + 2 * ns] >> 4; sc.Al = seg[3 + 2 * ns] & 15;
      sc.restart_interval = ri;
      // the tables start_pass_huff_decoder derives (jdhuff.c:95-135, jdphuff.c:95-200) must exist and be valid
      const bool prog = s->sof == 0xC2;
      const bool need_dc = !prog || (sc.Ss == 0 && sc.Ah == 0), need_ac = !prog || sc.Ss != 0;
      for (int i = 0; i < ns; i++) {
        if (need_dc && (sc.dc_huff[i] < 0 || derive_dec_table(s->huff[sc.dc_huff[i]], true, nullptr))) return bad(B200JPEG_ERR_BAD_SOURCE, "SOS names an undefined or bogus DC Huffman table");
        if (need_ac && (sc.ac_huff[i] < 0 || derive_dec_table(s->huff[sc.ac_huff[i]], false, nullptr))) return bad(B200JPEG_ERR_BAD_SOURCE, "SOS names an undefined or bogus AC Huffman table");
        const int ci = sc.component_index[i];
        if (!s->comp_quant_present[ci] && qdef[s->quant_tbl_no[ci]]) {                          // latch_quant_tables
          memcpy(s->comp_quant[ci], qcur[s->quant_tbl_no[ci]], sizeof qcur[0]); s->comp_quant_present[ci] = 1;
        }
      }
      saw_sos = true;
      sc.data_offset = pos + 2 + ln;
      const size_t end = scan_data_end(d, n, sc.data_offset);
      sc.data_size = end - sc.data_offset;
      s->num_scans++;
      pos = end;
      continue;
    } else {
      set_error("unknown JPEG marker 0x%02x", m);                                                // JERR_UNKNOWN_MARKER
      return B200JPEG_ERR_BAD_SOURCE;
    }
    pos += 2 + ln;
  }
  if (!saw_sof) return bad(B200JPEG_ERR_UNSUPPORTED, "only 1-, 3- and 4-component files are on the device path");
  const int nc = s->num_components;
  if (nc == 1) s->jpeg_color_space = B200JPEG_CS_GRAYSCALE;
  else if (nc == 3) {
    const bool ycc_ids = s->component_id[0] == 1 && s->component_id[1] == 2 && s->component_id[2] == 3;
    const bool rgb_ids = s->component_id[0] == 0x52 && s->component_id[1] == 0x47 && s->component_id[2] == 0x42;
    if (s->saw_JFIF) s->jpeg_color_space = B200JPEG_CS_YCbCr;
    else if (s->saw_Adobe) s->jpeg_color_space = s->Adobe_transform == 0 ? B200JPEG_CS_RGB : B200JPEG_CS_YCbCr;
    else if (ycc_ids) s->jpeg_color_space = B200JPEG_CS_YCbCr;
    else if (rgb_ids) s->jpeg_color_space = B200JPEG_CS_RGB;
    else s->jpeg_color_space = B200JPEG_CS_YCbCr;
  } else {
    s->jpeg_color_space = s->saw_Adobe && s->Adobe_transform == 2 ? B200JPEG_CS_YCCK : B200JPEG_CS_CMYK;
  }
  if (markers) {
    markers->clear();
    const bool multi = s->sof == 0xC2 || (s->num_scans && s->scans[0].comps_in_scan != nc);       // has_multiple_scans (jdinput.c)
    for (const Saved &m : saved)
      if (m.scans_seen == 0 || multi) markers->insert(markers->end(), d + m.pos, d + m.pos + m.len);
  }
  return B200JPEG_OK;
}

extern "C" int b200jpeg_parse_source(const uint8_t *d, size_t n, b200jpeg_source_info *s)
{
  return parse_source(d, n, s, nullptr);
}

// what default_decompress_parms (jdapimin.c:118-240) makes of the file's colour space
extern "C" int b200jpeg_decompress_output(const b200jpeg_source_info *src, int *width, int *height, int *color_space, int *components)
{
  if (!src || src->num_components < 1) return bad(B200JPEG_ERR_PARAM, "bad argument");
  const int cs = src->jpeg_color_space;
  if (width) *width = src->image_width;
  if (height) *height = src->image_height;
  if (color_space) *color_space = cs == B200JPEG_CS_GRAYSCALE ? B200JPEG_CS_GRAYSCALE : cs == B200JPEG_CS_YCbCr || cs == B200JPEG_CS_RGB ? B200JPEG_CS_RGB : B200JPEG_CS_CMYK;
  if (components) *components = src->num_components;
  return B200JPEG_OK;
}

extern "C" b200jpeg_decompress_options b200jpeg_default_decompress_options(void)
{
  b200jpeg_decompress_options o;
  o.scale_num = 1; o.scale_denom = 1; o.dct_method = B200JPEG_DCT_ISLOW; o.do_fancy_upsampling = 1; o.out_color_space = -1;
  return o;
}

namespace b200 {

// jpeg_calc_output_dimensions (jdmaster.c:96-370), the method choice of jddctmgr.c start_pass, jinit_upsampler
// (jdsample.c:421-530) and jinit_color_deconverter (jdcolor.c:760-930) for one source and one set of options
int plan_decompress(const b200jpeg_source_info &s, const b200jpeg_decompress_options &o, DecPlan &p)
{
  p = DecPlan();
  const int nc = s.num_components, jcs = s.jpeg_color_space;
  if (nc < 1 || nc > 4) return bad(B200JPEG_ERR_PARAM, "bad argument");
  if (o.scale_num < 1 || o.scale_denom < 1) { set_error("scale %d/%d: scale_num and scale_denom must be positive", o.scale_num, o.scale_denom); return B200JPEG_ERR_PARAM; }
  if (o.dct_method < B200JPEG_DCT_ISLOW || o.dct_method > B200JPEG_DCT_FLOAT) { set_error("dct_method %d is not JDCT_ISLOW, JDCT_IFAST or JDCT_FLOAT", o.dct_method); return B200JPEG_ERR_PARAM; }
  // the block size jpeg_core_output_dimensions picks: the least k with scale_num * 8 <= scale_denom * k, at most 16
  int k = 16;
  for (int t = 1; t < 16; t++) if ((long long)o.scale_num * 8 <= (long long)o.scale_denom * t) { k = t; break; }
  if (k != 1 && k != 2 && k != 4 && k != 8) {
    set_error("scale %d/%d gives an IDCT block size of %d: only sizes 1, 2, 4 and 8 (1/8, 1/4, 1/2, 1/1) are decoded on the device", o.scale_num, o.scale_denom, k);
    return B200JPEG_ERR_UNSUPPORTED;
  }
  p.k = k; p.method = o.dct_method;
  // out_color_space and the deconverter
  const int def = jcs == B200JPEG_CS_GRAYSCALE ? B200JPEG_CS_GRAYSCALE : jcs == B200JPEG_CS_YCbCr || jcs == B200JPEG_CS_RGB ? B200JPEG_CS_RGB : B200JPEG_CS_CMYK;
  const int ocs = o.out_color_space == -1 ? def : o.out_color_space;
  if (ocs < 0 || ocs > B200JPEG_CS_RGB565) { set_error("out_color_space %d is not a J_COLOR_SPACE", o.out_color_space); return B200JPEG_ERR_PARAM; }
  const bool refuse = ocs == B200JPEG_CS_RGB565 || ((ocs == B200JPEG_CS_CMYK || ocs == B200JPEG_CS_YCCK) && o.out_color_space != -1);
  if (refuse) { set_error("out_color_space %d (RGB565, CMYK or YCCK output) is not on the device path", ocs); return B200JPEG_ERR_UNSUPPORTED; }
  p.out_cs = ocs;
  bool conv_ok = true;
  if (ocs == B200JPEG_CS_GRAYSCALE) {
    p.out_nc = 1; p.ps = 1; p.nin = 1;
    if (jcs == B200JPEG_CS_GRAYSCALE || jcs == B200JPEG_CS_YCbCr) { p.conv = UPS_GRAY; for (int c = 1; c < nc; c++) p.needed[c] = false; }
    else if (jcs == B200JPEG_CS_RGB) { p.conv = UPS_RGB_GRAY; p.nin = 3; }
    else conv_ok = false;
  } else if (B200JPEG_CS_IS_RGB(ocs)) {
    p.out_nc = p.ps = B200JPEG_CS_PIXELSIZE(ocs);
    const int f = B200JPEG_CS_FIRST(ocs), bf = B200JPEG_CS_BLUE_FIRST(ocs);
    p.off[0] = f + (bf ? 2 : 0); p.off[1] = f + 1; p.off[2] = f + (bf ? 0 : 2); p.off[3] = f ? 0 : 3;
    if (jcs == B200JPEG_CS_YCbCr) { p.conv = UPS_YCC_RGB; p.nin = 3; }
    else if (jcs == B200JPEG_CS_GRAYSCALE) { p.conv = UPS_GRAY_RGB; p.nin = 1; }
    else if (jcs == B200JPEG_CS_RGB) { p.conv = UPS_COPY3; p.nin = 3; }
    else conv_ok = false;
  } else if (nc == 4 && ocs == B200JPEG_CS_CMYK) {         // the default of a CMYK / YCCK file (the batch refuses those)
    p.out_nc = p.ps = 4; p.nin = 0;
  } else if (ocs == jcs) {                                  // null_convert to the file's own space
    p.out_nc = p.ps = nc; p.nin = nc; p.conv = nc == 1 ? UPS_GRAY : UPS_COPY3;
    p.off[0] = 0; p.off[1] = 1; p.off[2] = 2;
  } else conv_ok = false;
  if (!conv_ok) return bad(B200JPEG_ERR_PARAM, "Unsupported color conversion request");   // JERR_CONVERSION_NOTIMPL
  // output size, and per component the IDCT size (chroma scaled up through the IDCT while that divides evenly) and
  // the downsampled size after scaling
  int mh = 1, mv = 1;
  for (int c = 0; c < nc; c++) { mh = std::max(mh, s.h_samp_factor[c]); mv = std::max(mv, s.v_samp_factor[c]); }
  const long long W = s.image_width, H = s.image_height;
  p.out_w = (int)((W * k + 7) / 8); p.out_h = (int)((H * k + 7) / 8);
  const bool do_fancy = o.do_fancy_upsampling && k > 1;
  for (int c = 0; c < nc; c++) {
    const int h = s.h_samp_factor[c], v = s.v_samp_factor[c];
    int ss = k;
    while (ss < 8 && (mh * k) % (h * ss * 2) == 0 && (mv * k) % (v * ss * 2) == 0) ss *= 2;
    p.ssize[c] = ss;
    p.dw[c] = (int)((W * h * ss + mh * 8 - 1) / (mh * 8)); p.dh[c] = (int)((H * v * ss + mv * 8 - 1) / (mv * 8));
    const int hin = h * ss / k, vin = v * ss / k;
    if (!hin || !vin || mh % hin || mv % vin || mh / hin > 2 || mv / vin > 2) { set_error("component %d: upsampling by %d x %d is not on the device path", c, mh / std::max(hin, 1), mv / std::max(vin, 1)); return B200JPEG_ERR_UNSUPPORTED; }
    p.hr[c] = mh / hin; p.vr[c] = mv / vin;
    // fancy: h2v1 / h2v2 need downsampled_width > 2, h1v2 does not; fullsize and int_upsample have no filter
    p.fancy[c] = do_fancy && (p.hr[c] == 2 ? p.dw[c] > 2 : p.vr[c] == 2);
  }
  p.is_default = k == 8 && p.method == B200JPEG_DCT_ISLOW && o.do_fancy_upsampling && ocs == def;
  return B200JPEG_OK;
}

}  // namespace b200

extern "C" int b200jpeg_decompress_output_opts(const b200jpeg_source_info *src, const b200jpeg_decompress_options *opts,
                                               int *width, int *height, int *color_space, int *components)
{
  if (!src || !opts || src->num_components < 1) return bad(B200JPEG_ERR_PARAM, "bad argument");
  DecPlan p;
  const int rc = plan_decompress(*src, *opts, p);
  if (rc) return rc;
  if (width) *width = p.out_w;
  if (height) *height = p.out_h;
  if (color_space) *color_space = p.out_cs;
  if (components) *components = p.out_nc;
  return B200JPEG_OK;
}

namespace b200 {

// The descriptors of a batch of sequential files (see decode.cuh).  The unstuffed words go to alloc(bound) first.
int build_decode_batch(const uint8_t *const *files, const size_t *sizes, int n, DecBatch &b, uint32_t *(*alloc)(void *, size_t), void *ctx, int first)
{
  if (b.want_markers) b.markers.resize(n);
  b.info.resize(n); b.scans.clear(); b.segs.clear(); b.tabs.clear();
  b.nsub = 0; b.nblocks = 0;
  size_t bound = 0;
  for (int i = 0; i < n; i++) {
    if (!files[i]) { set_error("image %d: no file", first + i); return B200JPEG_ERR_PARAM; }
    b200jpeg_source_info &s = b.info[i];
    int rc = parse_source(files[i], sizes[i], &s, b.want_markers ? &b.markers[i] : nullptr);
    if (rc) { std::string m = b200jpeg_last_error(); set_error("image %d: %s", first + i, m.c_str()); return rc; }
    if (s.sof == 0xC2) { set_error("image %d: progressive (SOF2) source: the device decode takes sequential files; pass its coefficients instead", first + i); return B200JPEG_ERR_UNSUPPORTED; }
    const b200jpeg_source_info &s0 = b.info[0];
    bool same = s.image_width == s0.image_width && s.image_height == s0.image_height && s.data_precision == s0.data_precision && s.num_components == s0.num_components;
    for (int c = 0; same && c < s.num_components; c++) same = s.h_samp_factor[c] == s0.h_samp_factor[c] && s.v_samp_factor[c] == s0.v_samp_factor[c];
    if (!same) { set_error("image %d: geometry (size, precision, components, sampling) differs from image 0", first + i); return B200JPEG_ERR_PARAM; }
  }
  const b200jpeg_source_info &s0 = b.info[0];
  b.W = s0.image_width; b.H = s0.image_height; b.nc = s0.num_components; b.precision = s0.data_precision;
  int hmax = 1, vmax = 1;
  for (int c = 0; c < b.nc; c++) { hmax = std::max(hmax, s0.h_samp_factor[c]); vmax = std::max(vmax, s0.v_samp_factor[c]); }
  for (int c = 0; c < b.nc; c++) {
    b.h[c] = s0.h_samp_factor[c]; b.v[c] = s0.v_samp_factor[c];
    b.wib[c] = (int)(((long long)b.W * b.h[c] + hmax * 8 - 1) / (hmax * 8));      // jdinput.c initial_setup
    b.hib[c] = (int)(((long long)b.H * b.v[c] + vmax * 8 - 1) / (vmax * 8));
  }
  auto scan_mcus = [&](const b200jpeg_source_scan &ss) -> long long {
    if (ss.comps_in_scan == 1) return (long long)b.wib[ss.component_index[0]] * b.hib[ss.component_index[0]];
    return (long long)((b.W + hmax * 8 - 1) / (hmax * 8)) * ((b.H + vmax * 8 - 1) / (vmax * 8));
  };
  for (int i = 0; i < n; i++)
    for (int k = 0; k < b.info[i].num_scans; k++) {
      const b200jpeg_source_scan &ss = b.info[i].scans[k];
      const long long ri = ss.restart_interval, nseg = ri ? (scan_mcus(ss) + ri - 1) / ri : 1;
      bound += ss.data_size + 16 * (size_t)nseg + 16;      // each segment: its bytes, up to 3 pad bytes, 2 zero words
    }
  uint32_t *out = alloc(ctx, bound / 4 + 4);
  if (!out) return B200JPEG_ERR_CUDA;
  unsigned long long wpos = 0;
  for (int i = 0; i < n; i++) {
    const b200jpeg_source_info &s = b.info[i];
    const uint8_t *d = files[i];
    std::map<int, int> tix;                          // pool index * 2 + is_dc -> DecTable index
    auto table = [&](int pool, bool dc) -> int {
      auto it = tix.find(pool * 2 + dc);
      if (it != tix.end()) return it->second;
      DecTable t; derive_dec_table(s.huff[pool], dc, &t);
      b.tabs.push_back(t); tix[pool * 2 + dc] = (int)b.tabs.size() - 1;
      return (int)b.tabs.size() - 1;
    };
    int scanned[4] = {0, 0, 0, 0};
    for (int k = 0; k < s.num_scans; k++) {
      const b200jpeg_source_scan &ss = s.scans[k];
      if (ss.Ss != 0 || ss.Se != 63 || ss.Ah != 0 || ss.Al != 0) { set_error("image %d: scan %d is not a sequential scan (Ss=%d Se=%d Ah=%d Al=%d)", first + i, k, ss.Ss, ss.Se, ss.Ah, ss.Al); return B200JPEG_ERR_BAD_SOURCE; }
      DecScan sc; memset(&sc, 0, sizeof sc);
      sc.img = i; sc.ncomp = ss.comps_in_scan;
      const long long mcus = scan_mcus(ss);
      sc.per_row = sc.ncomp == 1 ? b.wib[ss.component_index[0]] : (b.W + hmax * 8 - 1) / (hmax * 8);
      int slot = 0;
      for (int j = 0; j < sc.ncomp; j++) {
        const int c = ss.component_index[j];
        if (scanned[c]++) { set_error("image %d: component %d appears in two sequential scans", first + i, c); return B200JPEG_ERR_UNSUPPORTED; }
        const int hh = sc.ncomp == 1 ? 1 : b.h[c], vv = sc.ncomp == 1 ? 1 : b.v[c];
        sc.ci[j] = c; sc.first[j] = slot; sc.cnt[j] = hh * vv; sc.mx[c] = hh; sc.my[c] = vv;
        if (slot + hh * vv > 10) { set_error("image %d: scan %d has more than 10 blocks per MCU", first + i, k); return B200JPEG_ERR_BAD_SOURCE; }   // JERR_BAD_MCU_SIZE
        const int td = table(ss.dc_huff[j], true), ta = table(ss.ac_huff[j], false);
        for (int y = 0; y < vv; y++)
          for (int x = 0; x < hh; x++, slot++) { sc.comp[slot] = (int8_t)c; sc.dx[slot] = (int8_t)x; sc.dy[slot] = (int8_t)y; sc.tdc[slot] = (int16_t)td; sc.tac[slot] = (int16_t)ta; }
      }
      sc.nb = slot;
      const int scan_idx = (int)b.scans.size();
      b.scans.push_back(sc);
      // restart segments: unstuff into the upload buffer, one word-aligned stream per segment
      const int ri = ss.restart_interval;
      const long long nseg = ri ? (mcus + ri - 1) / ri : 1;
      size_t p = ss.data_offset; const size_t end = ss.data_offset + ss.data_size;
      for (long long sg = 0; sg < nseg; sg++) {
        uint8_t *o = reinterpret_cast<uint8_t *>(out + wpos);
        size_t cnt = 0;
        bool rst = false;
        while (p < end) {
          const uint8_t *f = static_cast<const uint8_t *>(memchr(d + p, 0xFF, end - p));
          const size_t q = f ? (size_t)(f - d) : end;
          memcpy(o + cnt, d + p, q - p); cnt += q - p; p = q;
          if (p >= end) break;
          size_t r = p + 1;
          while (r < end && d[r] == 0xFF) r++;                 // fill bytes
          if (r >= end) { p = end; break; }
          if (d[r] == 0x00) { o[cnt++] = 0xFF; p = r + 1; continue; }
          // RSTn (scan_data_end stops at every other marker)
          if (!ri) { set_error("image %d: scan %d: restart marker in a scan without restart interval", first + i, k); return B200JPEG_ERR_BAD_SOURCE; }
          if (d[r] - 0xD0 != (int)(sg & 7)) { set_error("image %d: scan %d: restart marker RST%d where RST%d was due", first + i, k, d[r] - 0xD0, (int)(sg & 7)); return B200JPEG_ERR_BAD_SOURCE; }
          p = r + 1; rst = true;
          break;
        }
        if (!rst && p >= end && sg + 1 < nseg) { set_error("image %d: scan %d ends after %lld of its %lld restart segments", first + i, k, sg + 1, nseg); return B200JPEG_ERR_BAD_SOURCE; }
        const size_t words = (cnt + 3) / 4 + 2;                // at least one zero word behind the data
        memset(o + cnt, 0, words * 4 - cnt);
        DecSeg g;
        g.word0 = wpos; g.nbits = (uint32_t)(cnt * 8); g.scan = scan_idx;
        g.mcu0 = (int)(sg * (ri ? ri : 0)); g.nmcu = (int)(ri ? std::min<long long>(ri, mcus - sg * ri) : mcus);
        g.sub0 = b.nsub; g.nsub = std::max(1, (int)((g.nbits + DEC_SUB_BITS - 1) / DEC_SUB_BITS));
        g.blk0 = b.nblocks;
        b.nsub += g.nsub; b.nblocks += (long long)g.nmcu * sc.nb;
        b.segs.push_back(g);
        wpos += words;
        if (cnt >= (1u << 29)) { set_error("image %d: a restart segment of 512 MB or more", first + i); return B200JPEG_ERR_UNSUPPORTED; }
      }
      // anything after the last segment's MCUs (further RSTn included) is ignored, like the reference
    }
  }
  b.nwords = wpos;
  return B200JPEG_OK;
}

}  // namespace b200
