// decode.cuh -- entropy decode of Huffman scans (jdhuff.c decode_mcu, jdphuff.c decode_mcu_*): the descriptors the
// host builds (source.cpp build_decode_batch) and the per-symbol step the decode kernels (kernels.cu) share.
//
// Each restart segment of a scan is an unstuffed bit stream starting on a word boundary of the batch's word buffer
// and followed by at least one zero word.  A decoder state is (zigzag index k within the block, 0 = at the block's
// start; block slot within the MCU), packed as k | slot << 7; DEC_DEAD marks a stream that hit an invalid code or ran
// out of bits.  Positions are bit offsets inside the segment.  The first scans of a coefficient (sequential, DC first,
// AC first) go through the speculative decode; the refinement scans of progressive files have kernels of their own.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define DEC_HD __host__ __device__ __forceinline__
#else
#define DEC_HD inline
#endif

namespace b200 {

#define DEC_DEAD 0xFFFFu
#define DEC_SUB_BITS 1024      // bits per speculatively decoded subsequence
#define DEC_CTA 128            // subsequences per CTA of the synchronisation kernel

// the colour conversions behind the decode with options (DecPlan::conv, k_upsample_opts): grayscale_convert,
// ycc_rgb_convert, null_convert / rgb_rgb_convert, gray_rgb_convert, rgb_gray_convert; for 4-component files
// ycck_cmyk_convert and null_convert (k_upsample_opts<4>)
enum { UPS_GRAY = 0, UPS_YCC_RGB = 1, UPS_COPY3 = 2, UPS_GRAY_RGB = 3, UPS_RGB_GRAY = 4, UPS_YCCK_CMYK = 5, UPS_COPY4 = 6 };

// jpeg_make_d_derived_tbl (jdhuff.c:143-261): 8-bit lookahead ((length << 8) | symbol, 0 = longer code), maxcode /
// valoffset per code length
struct DecTable { uint16_t look[256]; int32_t maxcode[18]; int32_t valoff[18]; uint8_t huffval[256]; };

// scan kinds: a sequential scan, and the four of a progressive file (jdphuff.c start_pass_phuff_decoder)
enum { DEC_SEQ = 0, DEC_DC_FIRST = 1, DEC_DC_REFINE = 2, DEC_AC_FIRST = 3, DEC_AC_REFINE = 4 };

// one scan of one image
struct DecScan {
  int img;                     // image inside the batch
  int kind, Ss, Se, Al;        // DEC_*; spectral band and point transform (0, 63, 0 for DEC_SEQ)
  int nb;                      // blocks per MCU
  int per_row;                 // MCUs per MCU row
  int ncomp;                   // components in the scan
  int ci[4], first[4], cnt[4]; // image component, first MCU slot and slots per MCU of scan component i
  int8_t comp[10], dx[10], dy[10];   // per MCU slot: image component, block offset inside the MCU
  int16_t tdc[10], tac[10];          // per MCU slot: DecTable index of its DC / AC table
  int mx[4], my[4];            // per image component: blocks per MCU across / down (1, 1 in a non-interleaved scan)
  long long base[4];           // per image component: first block of the image in the component's plane
  int wib[4], hib[4];          // per image component: its blocks across / down
};

// one restart segment (the whole scan without restarts)
struct DecSeg {
  unsigned long long word0;    // first word of the segment in the word buffer
  uint32_t nbits;              // unstuffed bits up to the next marker
  int scan;                    // DecScan index
  int mcu0, nmcu;              // MCUs of the scan this segment codes
  long long sub0;              // first subsequence (global index); segments are ordered by it
  int nsub;                    // subsequences, ceil(nbits / DEC_SUB_BITS) and at least 1
  long long blk0;              // first block in the DC-difference array (DC refinement: in the batch's refined blocks)
};

// per subsequence: the (position, state) its last decode started from and ended at, and the blocks it completed
struct DecRec { uint32_t in_pos, out_pos; uint32_t in_st, out_st; uint32_t count; uint32_t pad; };

// destination planes, one per component: each image's [hib][wib][64] int16 blocks, natural order, from the block
// DecScan::base gives (the per-image geometry is the scan's)
struct DecOut { int16_t *plane[4]; };

DEC_HD uint32_t dec_bswap(uint32_t x)
{
#if defined(__CUDA_ARCH__)
  return __byte_perm(x, 0, 0x0123);
#else
  return __builtin_bswap32(x);
#endif
}

// the 32 bits starting at bit `pos` of the big-endian stream w
DEC_HD uint32_t dec_window(const uint32_t *w, uint32_t pos)
{
  const uint32_t i = pos >> 5, sh = pos & 31;
  const unsigned long long v = ((unsigned long long)dec_bswap(w[i]) << 32) | dec_bswap(w[i + 1]);
  return (uint32_t)((v << sh) >> 32);
}

// The Huffman symbol at the top of win (jdhuff.c HUFF_DECODE): its code length, 0 for a code no table entry matches
DEC_HD int dec_symbol(uint32_t win, const DecTable &t, int &sym)
{
  const int look = t.look[win >> 24];
  if (look) { sym = look & 255; return look >> 8; }
  for (int l = 9; l <= 16; l++) {
    const int code = (int)(win >> (32 - l));
    if (code <= t.maxcode[l]) { sym = t.huffval[(code + t.valoff[l]) & 255]; return l; }
  }
  sym = 0;
  return 0;
}

// One Huffman symbol and its extra bits at `pos` in state `st` (decode_mcu, jdhuff.c:564-647; decode_mcu_DC_first and
// decode_mcu_AC_first, jdphuff.c:289-435).  Returns the next state, or DEC_DEAD (pos unchanged) for a code no table
// entry matches or a symbol that ends past nbits.  zz: the zigzag index the value goes to (0 = DC difference, -1 =
// none; a run past 63 writes index 63, like jpeg_natural_order's extra entries); done: the blocks the symbol ended,
// more than one for an EOB run of an AC first scan (the run is counted here and never becomes part of the state).
// PROG: the scan is a progressive first scan (DC first or AC first); the sequential instance keeps none of their cases
// in its per-symbol path.
template <bool PROG>
DEC_HD uint32_t dec_step(const uint32_t *w, uint32_t nbits, uint32_t &pos, uint32_t st, const DecScan &sc, const DecTable *tabs,
                         int &zz, int &val, int &done)
{
  zz = -1; val = 0; done = 0;                             // a dead stream completes no block
  int k = (int)(st & 127), slot = (int)(st >> 7);
  const bool acf = PROG && sc.kind == DEC_AC_FIRST;
  if (acf && k == 0) k = sc.Ss;
  const DecTable &t = tabs[k ? sc.tac[slot] : sc.tdc[slot]];
  const uint32_t win = dec_window(w, pos);
  int sym;
  const int len = dec_symbol(win, t, sym);
  if (!len) return DEC_DEAD;
  int s = k ? (sym & 15) : sym, r = k ? (sym >> 4) : 0;
  const bool eobr = acf && s == 0 && r != 15;             // EOBr: 2^r blocks plus r appended bits
  const int extra = eobr ? r : s;
  if ((unsigned long long)pos + (unsigned)(len + extra) > nbits) return DEC_DEAD;
  const int x = extra ? (int)((win << len) >> (32 - extra)) : 0;
  int v = 0;
  if (s) v = x < (1 << (s - 1)) ? x + (int)(~0u << s) + 1 : x;   // HUFF_EXTEND (jdhuff.c:483-490)
  pos += (uint32_t)(len + extra);
  val = v;
  if (k == 0) { zz = 0; k = PROG && sc.kind == DEC_DC_FIRST ? 64 : 1; }
  else if (s) { k += r; zz = k > 63 ? 63 : k; k++; }
  else if (r == 15) k += 16;
  else { k = 64; if (eobr) done = (1 << r) + x - 1; }
  if (k > (PROG ? sc.Se : 63)) { done++; k = 0; slot = slot + 1 == sc.nb ? 0 : slot + 1; }
  return (uint32_t)k | (uint32_t)slot << 7;
}

// decode from (pos, st) until pos reaches `end` or the stream dies; returns the blocks completed on the way
template <bool PROG>
DEC_HD uint32_t dec_run(const uint32_t *w, uint32_t nbits, uint32_t end, uint32_t &pos, uint32_t &st, const DecScan &sc, const DecTable *tabs)
{
  uint32_t n = 0;
  while (st != DEC_DEAD && pos < end) {
    int zz, val, done;
    const uint32_t ns = dec_step<PROG>(w, nbits, pos, st, sc, tabs, zz, val, done);
    st = ns; n += (uint32_t)done;
  }
  return n;
}

// dec_run with the instance for the scan's kind, chosen once per run
DEC_HD uint32_t dec_run(const uint32_t *w, uint32_t nbits, uint32_t end, uint32_t &pos, uint32_t &st, const DecScan &sc, const DecTable *tabs)
{
  return sc.kind == DEC_SEQ ? dec_run<false>(w, nbits, end, pos, st, sc, tabs) : dec_run<true>(w, nbits, end, pos, st, sc, tabs);
}

}  // namespace b200
