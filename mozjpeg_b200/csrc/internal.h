// internal.h -- shared declarations inside libb200jpeg (not installed).
#pragma once
#include "b200jpeg.h"
#include "decode.cuh"
#include <vector>
namespace b200 {
void set_error(const char *fmt, ...);
// lossless mode as the reference's validate_script detects it (jcmaster.c:302-311): the script's first entry has
// Ss != 0 and Se == 0 (the scan search skips the check, jcmaster.c:285-291)
bool is_lossless(const b200jpeg_params *p);
// the parameter block jpeg_start_compress works with in lossless mode (jcmaster.c:1072-1094): default colour space,
// 1x1 sampling, no smoothing, optimal tables; b200jpeg_enable_lossless's one-scan script follows the new component count
void lossless_start(const b200jpeg_params *in, b200jpeg_params *out);

// jpeg_make_d_derived_tbl with its validation (source.cpp); -1 for a table the reference refuses
int derive_dec_table(const b200jpeg_huff_tbl &h, bool is_dc, DecTable *out);
// start_pass_phuff_decoder's checks over every scan of a progressive file (jdphuff.c:91-144), with its warnings
// (JWRN_BOGUS_PROGRESSION) and a repeated first scan of a coefficient refused as well; coef_bits: [component][k], the
// point transform of the last scan that coded k (-1: none).  Messages name the scan, not the image.
int check_progression(const b200jpeg_source_info &s, int coef_bits[4][64]);
// smoothing_ok (jdcoefct.c:359-421) once the whole file is read: a decompress object at its defaults smooths the blocks
bool smoothing_applies(const b200jpeg_source_info &s, const int coef_bits[4][64]);
// one image's geometry (jdinput.c initial_setup): size, components, sampling factors, blocks across / down per
// component, and base[c]: where its blocks start in the batch's plane of component c (in blocks)
struct DecGeom {
  int W = 0, H = 0, nc = 0;
  int wib[4] = {0, 0, 0, 0}, hib[4] = {0, 0, 0, 0}, h[4] = {0, 0, 0, 0}, v[4] = {0, 0, 0, 0};
  long long base[4] = {0, 0, 0, 0};
};
// the host half of the device decode of a batch of files (source.cpp): parsed headers, per-image geometry, scan /
// segment descriptors, derived tables; the unstuffed segments go to the nwords words alloc(ctx, bound) returned.  segs:
// the segments of first scans (the speculative decode); dcr_segs: DC refinement segments (dcr_blocks blocks in all);
// acr_segs: AC refinement segments, level L (the L-th AC refinement scan of each image component) at
// [acr_level[L], acr_level[L + 1]).  Component c of every image lies in one plane of plane_blocks[c] blocks, the
// images' ranges one after another in batch order; a one-geometry batch is [n][hib][wib] blocks per component.
struct DecBatch {
  std::vector<b200jpeg_source_info> info;
  std::vector<DecScan> scans; std::vector<DecSeg> segs, dcr_segs, acr_segs; std::vector<DecTable> tabs;
  std::vector<int> acr_level;
  long long nsub = 0, nblocks = 0, dcr_blocks = 0; unsigned long long nwords = 0;
  // progressive: take SOF2 files (else they are refused as before)
  bool progressive = false;
  // mixed: take files of different geometry (else a file whose size, precision, components or sampling differ from
  // image 0's is refused)
  bool mixed = false;
  int precision = 8;
  std::vector<DecGeom> geom;
  long long plane_blocks[4] = {0, 0, 0, 0};
  // want_markers: also collect each file's COM / APPn segments as cjpeg copies them from a JPEG input (raw segments,
  // file order; see parse_source)
  bool want_markers = false;
  std::vector<std::vector<uint8_t>> markers;
};
// first: the batch index of files[0], for the messages (a caller that decodes a batch in chunks)
int build_decode_batch(const uint8_t *const *files, const size_t *sizes, int n, DecBatch &b, uint32_t *(*alloc)(void *, size_t), void *ctx, int first = 0);

// What jpeg_calc_output_dimensions, jinit_upsampler and jinit_color_deconverter decide for one source and one set of
// decompress options (source.cpp): output size and format, per component its DCT_scaled_size, downsampled size,
// replication factors after IDCT scaling and upsampler, whether it is needed at all, and the conversion (UPS_* of
// kernels.cuh) into ps bytes per pixel at off[].  is_default: the options give what a default decompress object gives.
struct DecPlan {
  int k = 8, method = 0, out_w = 0, out_h = 0, out_cs = 0, out_nc = 0;
  int ssize[4] = {8, 8, 8, 8}, dw[4] = {0, 0, 0, 0}, dh[4] = {0, 0, 0, 0}, hr[4] = {1, 1, 1, 1}, vr[4] = {1, 1, 1, 1};
  bool fancy[4] = {false, false, false, false}, needed[4] = {true, true, true, true};
  int conv = 0, nin = 1, ps = 1, off[4] = {0, 0, 0, 0};
  bool is_default = true;
};
int plan_decompress(const b200jpeg_source_info &s, const b200jpeg_decompress_options &o, DecPlan &p);

// What tj3DecompressToYUVPlanes8 (turbojpeg.c:2032-2195) decides for one source and one set of options (source.cpp):
// the TJSAMP_* getSubsamp assigns, the IDCT block size k every component runs (TurboJPEG overrides libjpeg's chroma
// scaling for TJSAMP_420), the IDCT method (B200JPEG_DCT_ISLOW or _IFAST), and per component the plane pw x ph, the
// IDCT output iw x ih and whether its table is the ifast multiplier table read by jpeg_idct_4x4 (int_table).
struct YuvPlan {
  int subsamp = -1, k = 8, method = 0, nc = 0, out_w = 0, out_h = 0;
  int pw[3] = {0, 0, 0}, ph[3] = {0, 0, 0}, iw[3] = {0, 0, 0}, ih[3] = {0, 0, 0};
  bool int_table[3] = {false, false, false};
};
int plan_yuv(const b200jpeg_source_info &s, const b200jpeg_decompress_options &o, YuvPlan &p);
}
