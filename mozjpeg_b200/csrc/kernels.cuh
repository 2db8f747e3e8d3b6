// kernels.cuh -- sm_90a device code of the JPEG-encode hot path.
//
// Everything here is integer / bit-serial or un-fused fp32 work: no tensor
// cores.  The file is compiled with -fmad=false because the trellis rate/
// distortion costs and the deringing filter must reproduce the reference's
// x86-64 (no FMA contraction) fp32 results bit for bit.
//
// Data layout in HBM (per batch of n images sharing one geometry):
//   coef[c] : int16 [n][hpad_c][wpad_c][64]   quantized coefficients, ZIGZAG order
//   raw[c]  : int16 [n][hpad_c][wpad_c][64]   FDCT output (x8 scale),  ZIGZAG order
// (one 128-byte line per 8x8 block; wpad/hpad include the dummy blocks that
// pad each component to whole interleaved MCUs, jccoefct.c:312-345).
// Sequential scans behind the default trellis additionally keep, per real block, a 128-byte symbol record and a dense
// int16 DC value (SymOut below): the entropy stages then read those, and coef[] keeps the plain-quantized values --
// except behind the tiled forward kernel (FwdStats), which counts the trellis statistics itself and writes no coef[]
// block; there coef[] holds only the blocks whose symbol record overflowed.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "decode.cuh"

namespace b200 {

// ---------------------------------------------------------------- geometry
struct CompGeom {
  int wib, hib;        // real blocks            (jcmaster.c:221-226)
  int wpad, hpad;      // incl. dummy blocks
  int h, v;            // sampling factors
  int hx, vx;          // hmax/h, vmax/v (downsampling box)
  int qt;              // quant table slot
  int dc_tbl, ac_tbl;  // Huffman table slots
  int rows_avail;      // downsampled rows holding real data (jcprepct.c:135-192)
  long long blocks_per_image;   // wpad*hpad
  int16_t *coef, *raw;
};
// restart parameters as the caller gave them (cinfo->restart_interval / restart_in_rows)
struct RestartSpec { int interval, in_rows; };
struct Geom {
  int W, H, nc, hmax, vmax;
  int mcus_per_row, mcu_rows;
  int in_comps;        // samples per input pixel
  int max_coef_bits;   // data_precision + 2
  int cs_mode;         // 0: RGB->YCbCr  1: RGB->gray  2: pass-through (sample ci of the pixel)  3: CMYK->YCCK
  int px_first, px_swap; // RGB-family pixel order (JCS_EXT_*): first colour sample inside the pixel, blue-first storage
  size_t row_pitch, image_stride;
  // raw-data input (jpeg_write_raw_data, jcapistd.c:145-195): downsampled component planes instead of pixels;
  // plane ci holds at least hib*8 rows of wib*8 samples; pitch and stride in bytes
  int raw_in;          // 1: sample planes; 2: quantized coefficient blocks (jpeg_write_coefficients), natural order
  const uint8_t *plane[4]; size_t plane_pitch[4], plane_stride[4];
  // per-image quantization: qset[img] (img counted inside the launch) is the index of the image's table set in the
  // QuantTables / TrellisConsts arrays the kernels receive; nullptr = every image uses set 0
  const int *qset;
  CompGeom c[4];
};
// the image's table set: base + qset[img]
template <class T> __device__ __forceinline__ const T *qset_of(const T *base, const Geom &g, int img) { return g.qset ? base + g.qset[img] : base; }

// component planes written by the input-smoothing pre-pass (pitch, stride in bytes)
struct PlanesOut { uint8_t *p[4]; size_t pitch[4], stride[4]; };

struct ScanDesc {
  int ncomps, ci[4];
  int Ss, Se, Ah, Al;
  int bim;                         // blocks per MCU in this scan
  int k_comp[10], k_y[10], k_x[10];
  int k_first[4], k_count[4];      // first k / number of blocks of scan-component i in the MCU
  int per_row, rows;               // MCUs per row / MCU rows of the scan (jcmaster.c:518-601)
  int ri;                          // restart interval of the scan in MCUs, 0 = none (jcmaster.c:594-599)
  const int *al_img;               // scan search: per-image Al replacing .Al (device pointer), or nullptr
  int dri;                         // scan search: this candidate's buffer starts with a DRI marker (its interval differs from the previous scan's)
  long long nblocks;               // per image
};

// quantizer constants per (table, natural index): exact floor((a + bias)/d)
// by multiply-shift (d = 8*Q, a < 2^18), see encoder.cu make_quant_consts().
// general form: q = ((|x| + bias) * mul) >> shift (64-bit product);  fast form (QuantTables.fast[t]): one shift
// L[t] for the whole table, q = umulhi((|x| + bias) << 14, mul2) >> L[t]  -- both exact for |x| + bias < 2^18.
struct QuantConst { uint32_t mul; uint16_t shift; uint16_t pad; uint32_t bias; uint32_t d; uint32_t mul2; };
// JDCT_IFAST: the scaled divisor's reciprocal / correction / shift (compute_reciprocal, jcdctmgr.c:181-230, DCTELEM = int)
struct IfastConst { uint32_t recip, corr; int shift; int pad; };
// qpack: {mul2, bias << 14} per natural position, the tiled forward kernel's shared copy of the fast quantizer
struct QuantTables { QuantConst q[4][64]; int L[4]; int fast[4]; float fdiv[4][64]; IfastConst ifast[4][64]; alignas(16) uint2 qpack[4][64]; };   // fdiv: JDCT_FLOAT divisors (jcdctmgr.c:355-379)                 // natural order
struct TrellisConsts {
  float w_zz[4][64];      // (float)(1.0/(Q*Q)) per zigzag position   jcdctmgr.c:1017-1021
  int   q8_zz[4][64];     // 8*Q per zigzag position
  unsigned qmul_zz[4][64]; int qL[4];          // exact a / q8 for a < 2^18: umulhi(a << 14, qmul_zz) >> qL (one shift per table)
  double p1, p2;          // pow(2, lambda_log_scale1), pow(2, lambda_log_scale2)
  float lambda_const;     // used when lambda_log_scale2 <= 0
  float delta_dc_weight;  // trellis_delta_dc_weight (jcdctmgr.c:1069-1086)
  int   use_norm;         // lambda_log_scale2 > 0
  int   max_coef_bits;    // data_precision + 2
  int   dc_trellis;       // trellis_quant_dc
  // the DC trellis' quantizer per table: (x + 4Q) / 8Q as an exact multiply-shift (like make_quant_consts), and whether
  // the table allows its FAST instantiation (9 candidates, no clamping reachable)
  unsigned dc_mul[4]; int dc_shift[4]; int dc_fast[4];
};

// Huffman table as the device keeps it: DHT payload + derived encode table.
struct DevHuff {
  uint8_t  bits[17];
  uint8_t  huffval[256];
  uint8_t  nsym;          // low 8 bits of the symbol count (count can be 256 -> see nsym16)
  uint8_t  pad0[12];
  uint16_t nsym16;
  uint16_t code[256];     // ehufco (jchuff.h:32-36)
  uint8_t  size[256];     // ehufsi; 0 = symbol has no code
};
static_assert(sizeof(DevHuff) == 17 + 256 + 1 + 12 + 2 + 512 + 256, "DevHuff layout");

// per real block side record: K1 writes {f = norm (jcdctmgr.c:1026-1030, before the /63),
// raw_dc, nz = number of non-zero plain-quantized AC coefficients, nzmask = their zigzag
// positions (bit i = position i, bit 0 clear)}; the band AC trellis (k_trellis_ac_band) replaces
// f by lambda_dc for the DC trellis, k_trellis_ac3 leaves it.
struct DcRec { float lambda_dc; int16_t raw_dc; uint8_t nz; uint8_t pad; unsigned long long nzmask; };
static_assert(sizeof(DcRec) == 16, "DcRec layout");
// where component ci's records start inside an image's record array
// sym_hi: byte offset of the symbol records' second plane (SYMREC_SPLIT below) = images in the chunk * per_image * 64
struct RecLayout { long long per_image; long long comp_off[4]; long long sym_hi; };
// which of the 8 table slots to (re)build for set i: m[i % period]
struct SlotMasks { uint32_t m[4]; int period; };

// Sequential scans after the AC trellis do not re-read the coefficient planes: the trellis back-track leaves, per real
// block (indexed like the side records), a symbol record -- word 0: number of entries (bit 7: more than SYMREC_SLOTS, the
// readers then walk the coefficient block), words 1..: one entry per AC symbol of the block, the stream's LAST symbol
// first, entry = run/size symbol | value bits << 16 (ZRL and EOB are entries too) -- and the DC trellis a dense array of
// the final DC values; `hist` (or nullptr) receives the blocks' AC symbol counts, [img][HIST_SLOTS][HIST_BINS].
#define SYMREC_BYTES 128
#define SYMREC_SLOTS 31
// SYMREC_SPLIT: a record lives in two 64-byte halves, words 0..15 in plane 0 and words 16..31 in plane 1 (both indexed like
// the side records), instead of one 128-byte slot: the readers fetch the header and the first entries of every block, and
// L2 fills whole 128-byte lines -- with one slot per line the bit-count and packing kernels moved 26 / 28 MB per 4K image
// for ~8 MB of entries; with two blocks per line the second plane is touched only by blocks of 16 and more symbols.
#ifndef SYMREC_SPLIT
#define SYMREC_SPLIT 1
#endif
// keep_coef: also rewrite the coefficient planes (the debug tap reads them); otherwise only blocks whose record overflowed
// get their coefficients written back, and the planes keep the plain-quantized values elsewhere.
// dcq_ac: the AC trellis fills dcq with the plain-quantized DC values (no DC trellis will follow and write the final ones).
struct SymOut { uint8_t *sym; int16_t *dcq; uint32_t *hist; int keep_coef; int dcq_ac; };

#define HIST_BINS 257
#define HIST_SLOTS 8          // [is_ac*4 + tbl_no]

// ---------------------------------------------------------------- launches (defined in kernels.cu)
// status[img] bits: 2 = JERR_BAD_DCT_COEF / missing Huffman code, 4 = output buffer too small (host retries)
// the raw DCT plane is written only when the trellis (rec != nullptr) or the debug tap (keep_raw) will read it
// qt / tc (here and in the trellis launches): the batch's table sets, image img reads set g.qset[img] (qset_of);
// qfast / dc_fast: every set the launch's images use allows the fast form
void launch_prep_planes(const Geom &g, const uint8_t *src, int smoothing_factor, const PlanesOut &out, int n, cudaStream_t s);
// TurboJPEG YUV planes (k_encode_yuv): plane ci of image img starts at p[ci] + img * stride[ci] and holds ph[ci] rows of
// pw[ci] samples pitch[ci] bytes apart (b200jpeg_yuv_plane_dims); g.hmax, g.vmax in {1, 2, 4}, component 0 at them and
// components 1, 2 (g.nc == 3) 1x1; 8-bit samples
struct YuvOut { uint8_t *p[3]; size_t pitch[3], stride[3]; int pw[3], ph[3]; };
void launch_encode_yuv(const Geom &g, const uint8_t *src, const YuvOut &out, int n, cudaStream_t s);
// raw_in == 2: planes hold JBLOCK rows.  xf: the block mapping of a lossless transform (b200jpeg_transform_info, per
// component; all zero = the plain copy): the planes are then in the source's geometry, pitch and stride
struct CoefXform { int transposed; int x_crop[4], y_crop[4], x_mirror[4], y_mirror[4]; };
void launch_import_coefs(const Geom &g, const CoefXform &xf, int n, cudaStream_t s);
// Trellis-phase statistics counted by the tiled forward kernel (fs.hist != nullptr, only where forward_tiled() holds):
// every real block's AC symbols go into hist [img*nc + ci][4 + ac_tbl][sym] (zeroed by the caller), its plain-quantized
// DC into dcq (indexed like the side records), JERR_BAD_DCT_COEF into status; the coefficient planes are not written
struct FwdStats { uint32_t *hist; int16_t *dcq; uint32_t *status; };
bool forward_tiled(const Geom &g, int dct_method);   // launch_forward runs k_forward_tile for this geometry
void launch_forward(const Geom &g, const uint8_t *src, const QuantTables *qt, int qfast, int dct_method /* J_DCT_METHOD */, int dering, DcRec *rec, const RecLayout &rl, int keep_raw,
                    const FwdStats &fs, int n, cudaStream_t s);
void launch_dummy(const Geom &g, int n, cudaStream_t s);
void launch_gather_comp(const Geom &g, const RestartSpec &rs, uint32_t *hist, uint32_t *status, int n, cudaStream_t s);
// the DC half of the trellis-phase statistics from the dense DC values (the AC half came from the forward kernel)
void launch_gather_comp_dc(const Geom &g, const RestartSpec &rs, const int16_t *dcq, const RecLayout &rl, uint32_t *hist, uint32_t *status, int n, cudaStream_t s);
// nz_rec (here and in launch_block_bits / launch_encode): the side records holding every block's final non-zero positions
// (trellis on, sequential scans), or nullptr
void launch_gather_seq(const Geom &g, const ScanDesc &sd, const DcRec *nz_rec, const uint8_t *sym, const int16_t *dcq, const RecLayout &rl, uint32_t *hist, uint32_t *status, int n, cudaStream_t s);
void launch_seed_hist(uint32_t *hist, int slot, int n, cudaStream_t s);
void launch_gen_tables(const uint32_t *hist, DevHuff *tabs, size_t tabs_set_stride, const SlotMasks &masks, int nsets, cudaStream_t s);
// AC trellis of the default option set: launch_trellis_sort sorts the side records by non-zero count (srec: 16 bytes
// per real block; splits: 4 class boundaries per (image, component) followed by 128 words of sorting counters each),
// then launch_trellis_ac3 runs one class-specific kernel per count class.  The records keep the forward kernel's norm
// (the DC trellis behind it derives lambda_dc: launch_trellis_dc with lambda_from_norm)
void launch_trellis_sort(const Geom &g, const DcRec *rec, const RecLayout &rl, void *srec, uint32_t *splits, int n, cudaStream_t s);
void launch_trellis_ac3(const Geom &g, const TrellisConsts *tc, const DevHuff *tabs, size_t tabs_set_stride,
                        DcRec *rec, const RecLayout &rl, const void *srec, const uint32_t *splits, const SymOut &so, int n, int sms, cudaStream_t s);
// use_scans_in_trellis: quantize_trellis restricted to the zigzag band [Ss, Se]
void launch_trellis_ac_band(const Geom &g, const TrellisConsts *tc, const DevHuff *tabs, size_t tabs_set_stride,
                            DcRec *rec, const RecLayout &rl, int Ss, int Se, const uint16_t *qimg, float4 *eo, int n, cudaStream_t s);
// trellis_eob_opt: block-level EOB-run pass over every block row (eo from the band kernel; scratch: 16 bytes per real block)
void launch_trellis_eob_rows(const Geom &g, const DevHuff *tabs, size_t tabs_set_stride, DcRec *rec, const RecLayout &rl, int Ss, int Se,
                             const float4 *eo, void *scratch, int n, cudaStream_t s);
// trellis_q_opt: accumulate the table-fitting sums of the components in g ([img][4][2][64] int64) / re-fit the per-image tables
void launch_qopt_sums(const Geom &g, long long *qsum, int n, cudaStream_t s);
void launch_qopt_update(long long *qsum, uint16_t *qimg, int n, cudaStream_t s);
// dcq (or nullptr): dense array of the final DC values, one per real block, indexed like the side records; with it and
// write_coef == 0 the coefficient planes are not touched.  vertical: trellis_delta_dc_weight > 0.  lambda_from_norm:
// the records hold the forward kernel's norm (behind launch_trellis_ac3), not lambda_dc (behind launch_trellis_ac_band)
void launch_trellis_dc(const Geom &g, const TrellisConsts *tc, const DevHuff *tabs, size_t tabs_set_stride,
                       const DcRec *rec, const RecLayout &rl, int vertical, int dc_fast, int16_t *dcq, int write_coef,
                       int lambda_from_norm, int n, cudaStream_t s);
// DC statistics of a sequential scan from the dense DC array (+ the EOB of every dummy block): with the AC counts the
// trellis back-track left in `hist`, the scan's complete statistics (encode_mcu_gather, jchuff.c:886-915)
void launch_gather_seq_dc(const Geom &g, const ScanDesc &sd, const int16_t *dcq, const RecLayout &rl, uint32_t *hist, uint32_t *status, int n, cudaStream_t s);
// tile_last / tile_first: int [n][ceil(nblocks/256)] scratch; pm: the blocks' event masks of this AC scan,
// unsigned long long [3][n][nblocks] (written here, read by the three symbol walks of the scan)
void launch_prog_prepare(const Geom &g, const ScanDesc &sd, uint32_t *aux, uint32_t *run_e, unsigned long long *pm, int *tile_last, int *tile_first, int n, cudaStream_t s);
void launch_gather_prog(const Geom &g, const ScanDesc &sd, const uint32_t *aux, const uint32_t *run_e, const unsigned long long *pm, uint32_t *hist, uint32_t *status, int n, cudaStream_t s);
// sym / dcq (here and in launch_encode): the symbol records and dense DC values of sequential scans after the trellis, or nullptr
void launch_block_bits(const Geom &g, const ScanDesc &sd, const DcRec *nz_rec, const uint8_t *sym, const int16_t *dcq, const RecLayout &rl, const DevHuff *tabs, size_t tabs_image_stride, int progressive,
                       uint32_t *blk_bits, uint32_t *tile_bits, const uint32_t *blk_aux, const uint32_t *run_e, const unsigned long long *pm, uint32_t *status, int n, cudaStream_t s);
// tile_base[img][tile] / seg_corr[img][segment] / total_bits[img] from the tile sums (and the restart interval)
void launch_scan_layout(const ScanDesc &sd, const uint32_t *blk_bits, const uint32_t *tile_bits, unsigned long long *tile_base,
                        uint32_t *seg_corr, long long seg_stride, unsigned long long *total_bits, size_t capacity_bits,
                        uint32_t *status, int n, cudaStream_t s);
// clears the part of every image's word stream that the scan laid out by launch_scan_layout will occupy
void launch_zero_stream(uint32_t *bitbuf, size_t bitbuf_image_stride_words, const unsigned long long *total_bits, int n, cudaStream_t s);
// mark: bitmap over the unstuffed bytes of each image (restart markers' 0xFF), only touched when sd.ri != 0
// nz_rec: the side records holding every block's final non-zero positions (trellis on, sequential scans), or nullptr
void launch_encode(const Geom &g, const ScanDesc &sd, const DcRec *nz_rec, const uint8_t *sym, const int16_t *dcq, const RecLayout &rl, const DevHuff *tabs, size_t tabs_image_stride, int progressive,
                   const uint32_t *blk_bits, const uint32_t *tile_bits, const unsigned long long *tile_base, const uint32_t *seg_corr, long long seg_stride,
                   const uint32_t *blk_aux, const uint32_t *run_e, const unsigned long long *pm,
                   uint32_t *bitbuf, size_t bitbuf_image_stride_words, uint32_t *mark, size_t mark_stride_words, const uint32_t *status, int n, cudaStream_t s);
// byte stuffing of every scan in one pass with a decoupled look-back (k_stuff): out[img][out_start[img] ...], scan_size,
// out_next.  lookback: stuff_lookback_bytes() of look-back state (a descriptor per tile, a ticket per image), all zero
// before each launch.
size_t stuff_tiles(size_t bitbuf_image_stride_words);
size_t stuff_lookback_bytes(size_t bitbuf_image_stride_words, int n);
void launch_stuff(const uint32_t *bitbuf, size_t bitbuf_image_stride_words, const unsigned long long *total_bits, void *lookback,
                  uint8_t *out, size_t out_image_stride, size_t out_capacity, const unsigned long long *out_start, unsigned long long *out_next,
                  uint32_t *scan_size, uint32_t *status, const uint32_t *mark, size_t mark_stride_words, int n, cudaStream_t s);

// lossless (SOF3) scans: sd.ncomps components of one sample per MCU, sd.nblocks = W*H MCUs, sd.Ss the predictor, sd.Al
// the point transform, sd.ri the restart interval in MCUs (whole rows).  diff: [n][sd.ncomps][W*H] uint16 differences
// (mod 2^16); hist: the categories per DC table, [img][HIST_SLOTS][HIST_BINS] (zeroed by the caller).  The bit counts,
// layout, packing and stuffing follow the sequential scans' stages (launch_scan_layout, launch_zero_stream, launch_stuff).
void launch_lossless_diff(const Geom &g, const ScanDesc &sd, int precision, const uint8_t *src, uint16_t *diff, uint32_t *hist, int n, cudaStream_t s);
void launch_lossless_bits(const Geom &g, const ScanDesc &sd, const uint16_t *diff, const DevHuff *tabs, size_t tabs_image_stride,
                          uint32_t *blk_bits, uint32_t *tile_bits, uint32_t *status, int n, cudaStream_t s);
void launch_lossless_encode(const Geom &g, const ScanDesc &sd, const uint16_t *diff, const DevHuff *tabs, size_t tabs_image_stride,
                            const uint32_t *blk_bits, const unsigned long long *tile_base, const uint32_t *seg_corr, long long seg_stride,
                            uint32_t *bitbuf, size_t bitbuf_image_stride_words, uint32_t *mark, size_t mark_stride_words, const uint32_t *status, int n, cudaStream_t s);

// scan search: per-image best point transform of one Al-search group (see k_select_al)
struct AlSearch { ScanDesc sd[24]; int first, per_al, nband, al_max, nscans_total; };
void launch_select_al(const Geom &g, const AlSearch &as, const DevHuff *tabs_scan, const uint32_t *scan_size, int n, int *best_al, cudaStream_t s);

// sequential Huffman decode (decode.cuh): k_dec_sync, k_dec_fix, the block-count scan, k_dec_write, k_dec_dc on the
// batch's descriptors; rec: nsub records, pre: nsub words, tsum: ceil(nsub / 1024) words, dcd: one int per block of
// every scan (dummy blocks included); o: the destination in device memory; the planes are zeroed by the caller; status[img] bit 0 = corrupt data;
// max_rounds / redone: synchronisation work (zeroed by the caller); marks: 6 events recorded around the stages
void launch_decode(const uint32_t *words, const DecSeg *segs, int nsegs, const DecScan *scans, const DecTable *tabs, long long nsub,
                   DecRec *rec, uint32_t *pre, unsigned long long *tsum, int *dcd, const DecOut *o, uint32_t *status,
                   int *max_rounds, unsigned long long *redone, cudaEvent_t *marks, cudaStream_t s);

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
// multiplier tables), 2 k_idct_float (tab: float multiplier tables); image i's table at tab + i * qstride entries.
// out: [n][hib * size][wib * size] samples.
void launch_idct_opts(int size, int method, const int16_t *coef, const void *tab, int qstride, uint8_t *out, int wib, int hib, int n, cudaStream_t s);
// k_upsample_opts: per used component (nin of them) image 0's plane, pitch / stride in bytes, dw x dh real samples,
// the replication factors hr x vr (1 or 2) after IDCT scaling, and fancy (the smoothing filter instead of
// replication); conv the colour conversion (UPS_* of decode.cuh); ps bytes per pixel with R, G, B (or the one gray byte) at off[0..2] and
// 0xFF at off[3] when ps is 4.
struct UpsOpt {
  const uint8_t *plane[3]; int pitch[3]; long long stride[3]; int dw[3], dh[3], hr[3], vr[3], fancy[3];
  int nin, conv, ps, off[4];
};
void launch_upsample_opts(const UpsOpt &o, uint8_t *pix, size_t row_pitch, size_t image_stride, int W, int H, int n, cudaStream_t s);

extern unsigned long long g_kernel_launches;

}  // namespace b200
