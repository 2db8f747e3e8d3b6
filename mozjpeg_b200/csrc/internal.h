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
// the host half of the device decode of a batch of sequential files (source.cpp): parsed headers, one geometry,
// scan / segment descriptors, derived tables; the unstuffed segments go to the nwords words alloc(ctx, bound) returned
struct DecBatch {
  std::vector<b200jpeg_source_info> info;
  std::vector<DecScan> scans; std::vector<DecSeg> segs; std::vector<DecTable> tabs;
  long long nsub = 0, nblocks = 0; unsigned long long nwords = 0;
  int W = 0, H = 0, nc = 0, precision = 8;
  int wib[4] = {0, 0, 0, 0}, hib[4] = {0, 0, 0, 0}, h[4] = {0, 0, 0, 0}, v[4] = {0, 0, 0, 0};
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
}
