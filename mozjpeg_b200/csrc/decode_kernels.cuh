// decode_kernels.cuh -- sm_90a device code of the JPEG decompressor: the entropy decode of the first and refinement
// scans, the IDCTs, the upsamplers and colour conversions (decode_kernels.cu, compiled with -fmad=false like kernels.cu:
// k_idct_float must reproduce the reference's fp32 results without FMA contraction).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "decode.cuh"

namespace b200 {

// Huffman decode of the first scans (decode.cuh): k_dec_sync, k_dec_fix, the block-count scan, k_dec_write, k_dec_dc on
// the batch's descriptors; rec: nsub records, pre: nsub words, tsum: ceil(nsub / 1024) words, dcd: one int per block of
// every scan (dummy blocks included); o: the destination in device memory; the planes are zeroed by the caller; status[img] bit 0 = corrupt data, bit 1 = a
// coefficient past its band;
// max_rounds / redone: synchronisation work (zeroed by the caller); marks: 6 events recorded around the stages
void launch_decode(const uint32_t *words, const DecSeg *segs, int nsegs, const DecScan *scans, const DecTable *tabs, long long nsub,
                   DecRec *rec, uint32_t *pre, unsigned long long *tsum, int *dcd, const DecOut *o, uint32_t *status,
                   int *max_rounds, unsigned long long *redone, cudaEvent_t *marks, cudaStream_t s);

// the refinement scans of progressive files, after launch_decode: k_dec_dc_refine over the dcr_blocks blocks of the ndcr
// DC refinement segments, then k_dec_ac_refine once per level over AC refinement segments [acr_level[l],
// acr_level[l + 1]) (acr_level: host memory); status[img]: bit 0 corrupt data or too few bits, bit 1 a coefficient past
// its band, bit 2 a refinement symbol of size other than 1; marks: 2 events recorded behind the two stages
void launch_decode_refine(const uint32_t *words, const DecSeg *dcr, int ndcr, long long dcr_blocks, const DecSeg *acr, const int *acr_level, int nlevels,
                          const DecScan *scans, const DecTable *tabs, const DecOut *o, uint32_t *status, cudaEvent_t *marks, cudaStream_t s);

// decompression to pixels behind the entropy decode (jpeg_read_scanlines of a default decompress object, 8-bit).
// k_idct_islow: coef [n][hib][wib][64] natural order -> out [n][hib * 8][wib * 8] samples, dequantized with image i's
// table (natural order) at quant + i * qstride.
void launch_idct_islow(const int16_t *coef, const uint16_t *quant, int qstride, uint8_t *out, int wib, int hib, int n, cudaStream_t s);
// k_upsample_color<hx, vx, nc>: the sample planes (image 0's, pitch / stride in bytes; planes 1 and 2 share theirs and
// hold dw x dh real samples) -> W x H interleaved pixels of nc samples; hx, vx: luma over chroma sampling, 1 or 2 each;
// ycc: convert YCbCr to RGB, else copy the components.  Returns -1 for a layout it has no kernel for.
int launch_upsample_color(int hx, int vx, int nc, const uint8_t *const *planes, const int *pitch, const long long *stride, int dw, int dh, bool ycc,
                          uint8_t *pix, size_t row_pitch, size_t image_stride, int W, int H, int n, cudaStream_t s);

// decompression with options.  IDCT of one component whose DCT_scaled_size is `size`: 1, 2, 4 -> k_idct_red<size>
// (tab: the uint16 quantization tables), 8 -> by method: 0 islow (tab as for 1 .. 4), 1 k_idct_ifast (tab: int
// multiplier tables), 2 k_idct_float (tab: float multiplier tables); 3, 5, 6, 7 and 9 .. 16 -> k_idct_scaled<size>
// whatever the method (tab as for 1 .. 4: jddctmgr.c gives those sizes the islow-style table); image i's table at
// tab + i * qstride entries.  out: [n][hib * size][wib * size] samples.
void launch_idct_opts(int size, int method, const int16_t *coef, const void *tab, int qstride, uint8_t *out, int wib, int hib, int n, cudaStream_t s);
// k_upsample_opts<NC>: per used component (nin of them) image 0's plane, pitch / stride in bytes, dw x dh real samples,
// the replication factors hr x vr (1 or 2) after IDCT scaling, and fancy (the smoothing filter instead of
// replication); conv the colour conversion (UPS_* of decode.cuh).  NC = 3 (UpsOpt): 1- and 3-component files, ps bytes
// per pixel with R, G, B (or the one gray byte) at off[0..2] and 0xFF at off[3] when ps is 4.  NC = 4 (UpsOpt4):
// 4-component files, conv UPS_YCCK_CMYK or UPS_COPY4, 4 bytes a pixel in component order (ps and off unused).
template <int NC> struct UpsOptN {
  const uint8_t *plane[NC]; int pitch[NC]; long long stride[NC]; int dw[NC], dh[NC], hr[NC], vr[NC], fancy[NC];
  int nin, conv, ps, off[4];
};
typedef UpsOptN<3> UpsOpt;
typedef UpsOptN<4> UpsOpt4;
template <int NC>
void launch_upsample_opts(const UpsOptN<NC> &o, uint8_t *pix, size_t row_pitch, size_t image_stride, int W, int H, int n, cudaStream_t s);

// The pixel stage of a chunk whose images differ in geometry: the same kernels driven by a work table, one 4-byte image
// index per CTA, and a descriptor per image.  An IDCT image: wib x hib blocks from block `coef` of the coefficient
// plane, its table at `tab` entries, its samples at byte `out`, wib * size a row; cta0: its first CTA, its blocks
// padded to whole CTAs of idct_blocks_per_cta(size) blocks.  size and method as for launch_idct_opts.
struct IdctImg { long long coef, out; int wib, hib, tab, cta0; };
int idct_blocks_per_cta(int size);
void launch_idct_ragged(int size, int method, const int16_t *coef, const void *tab, uint8_t *out, const uint32_t *work, const IdctImg *imgs,
                        unsigned ncta, cudaStream_t s);
// An upsampling / colour conversion image: its UpsOpt (planes of its own; stride unused), W x H pixels at pix,
// row_pitch bytes apart; cta0: its first CTA, gx: its 64 x 4 pixel tiles a row.
template <int NC> struct UpsImgN { UpsOptN<NC> o; uint8_t *pix; long long row_pitch; int W, H, cta0, gx; };
typedef UpsImgN<3> UpsImg;
typedef UpsImgN<4> UpsImg4;
template <int NC>
void launch_upsample_ragged(const uint32_t *work, const UpsImgN<NC> *imgs, unsigned ncta, cudaStream_t s);

// Decompression to YUV planes (jpeg_read_raw_data): the IDCT kernels above with their PLANE store, which writes image
// i's samples straight into out + i * stride, rows `pitch` bytes apart, clipped to the first cw columns and ch rows.
// size as for launch_idct_opts, method 0 (islow) or 1 (ifast: tab as for launch_idct_opts); int_table: size 4 reading an int table (tab as for method 1) the way
// jpeg_idct_4x4 reads its islow table, which is what a TJSAMP_420 chroma component gets at 1/2 with JDCT_IFAST.
struct IdctDst { long long pitch, stride; int cw, ch; };
// Decoding YUV planes to pixels (tj3DecodeYUVPlanes8, do_fancy_upsampling off): pixel (x, y) of image i from luma
// sample (x, y) and chroma sample (x >> hs, y >> vs) of image i's planes (plane[c] + i * stride[c], pitch[c] bytes a
// row); conv UPS_GRAY (luma only), UPS_GRAY_RGB or UPS_YCC_RGB; ps bytes a pixel with R, G, B at off[0..2] and 0xFF at
// off[3] when ps is 4.
struct YuvPix { const uint8_t *plane[3]; long long pitch[3], stride[3]; int hs, vs, conv, ps, off[4]; };
void launch_yuv_to_pixels(const YuvPix &d, uint8_t *pix, size_t row_pitch, size_t image_stride, int W, int H, int n, cudaStream_t s);
void launch_idct_plane(int size, int method, bool int_table, const int16_t *coef, const void *tab, int qstride, uint8_t *out, const IdctDst &d,
                       int wib, int hib, int n, cudaStream_t s);

}  // namespace b200
