// decode.cuh -- entropy decode of sequential Huffman scans (jdhuff.c decode_mcu): the descriptors the host builds
// (source.cpp build_decode_batch) and the per-symbol step the decode kernels (kernels.cu) share.
//
// Each restart segment of a scan is an unstuffed bit stream starting on a word boundary of the batch's word buffer
// and followed by at least one zero word.  A decoder state is (zigzag index k within the block, 0 = expecting the DC
// difference; block slot within the MCU), packed as k | slot << 7; DEC_DEAD marks a stream that hit an invalid code
// or ran out of bits.  Positions are bit offsets inside the segment.
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
// ycc_rgb_convert, null_convert / rgb_rgb_convert, gray_rgb_convert, rgb_gray_convert
enum { UPS_GRAY = 0, UPS_YCC_RGB = 1, UPS_COPY3 = 2, UPS_GRAY_RGB = 3, UPS_RGB_GRAY = 4 };

// jpeg_make_d_derived_tbl (jdhuff.c:143-261): 8-bit lookahead ((length << 8) | symbol, 0 = longer code), maxcode /
// valoffset per code length
struct DecTable { uint16_t look[256]; int32_t maxcode[18]; int32_t valoff[18]; uint8_t huffval[256]; };

// one scan of one image
struct DecScan {
  int img;                     // image inside the batch
  int nb;                      // blocks per MCU
  int per_row;                 // MCUs per MCU row
  int ncomp;                   // components in the scan
  int ci[4], first[4], cnt[4]; // image component, first MCU slot and slots per MCU of scan component i
  int8_t comp[10], dx[10], dy[10];   // per MCU slot: image component, block offset inside the MCU
  int16_t tdc[10], tac[10];          // per MCU slot: DecTable index of its DC / AC table
  int mx[4], my[4];            // per image component: blocks per MCU across / down (1, 1 in a non-interleaved scan)
};

// one restart segment (the whole scan without restarts)
struct DecSeg {
  unsigned long long word0;    // first word of the segment in the word buffer
  uint32_t nbits;              // unstuffed bits up to the next marker
  int scan;                    // DecScan index
  int mcu0, nmcu;              // MCUs of the scan this segment codes
  long long sub0;              // first subsequence (global index); segments are ordered by it
  int nsub;                    // subsequences, ceil(nbits / DEC_SUB_BITS) and at least 1
  long long blk0;              // first block in the DC-difference array
};

// per subsequence: the (position, state) its last decode started from and ended at, and the blocks it completed
struct DecRec { uint32_t in_pos, out_pos; uint32_t in_st, out_st; uint32_t count; uint32_t pad; };

// destination planes: [n][hib][wib][64] int16 per component, natural order
struct DecOut { int16_t *plane[4]; int wib[4], hib[4]; };

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

// One Huffman symbol and its extra bits at `pos` in state `st` (decode_mcu, jdhuff.c:564-647).  Returns the next state,
// or DEC_DEAD (pos unchanged) for a code no table entry matches or a symbol that ends past nbits.  zz: the zigzag index
// the value goes to (0 = DC difference, -1 = none; a run past 63 writes index 63, like jpeg_natural_order's extra
// entries); done: the symbol ended its block.
DEC_HD uint32_t dec_step(const uint32_t *w, uint32_t nbits, uint32_t &pos, uint32_t st, const DecScan &sc, const DecTable *tabs,
                         int &zz, int &val, bool &done)
{
  int k = (int)(st & 127), slot = (int)(st >> 7);
  const DecTable &t = tabs[k ? sc.tac[slot] : sc.tdc[slot]];
  const uint32_t win = dec_window(w, pos);
  int len, sym;
  const int look = t.look[win >> 24];
  if (look) { len = look >> 8; sym = look & 255; }
  else {
    len = 0; sym = 0;
    for (int l = 9; l <= 16; l++) {
      const int code = (int)(win >> (32 - l));
      if (code <= t.maxcode[l]) { len = l; sym = t.huffval[(code + t.valoff[l]) & 255]; break; }
    }
    if (!len) return DEC_DEAD;
  }
  const int s = k ? (sym & 15) : sym, r = k ? (sym >> 4) : 0;
  if ((unsigned long long)pos + (unsigned)(len + s) > nbits) return DEC_DEAD;
  int v = 0;
  if (s) {
    const int x = (int)((win << len) >> (32 - s));
    v = x < (1 << (s - 1)) ? x + (int)(~0u << s) + 1 : x;          // HUFF_EXTEND (jdhuff.c:483-490)
  }
  pos += (uint32_t)(len + s);
  zz = -1; val = v; done = false;
  if (k == 0) { zz = 0; k = 1; }
  else if (s) { k += r; zz = k > 63 ? 63 : k; k++; }
  else if (r == 15) k += 16;
  else k = 64;
  if (k >= 64) { done = true; k = 0; slot = slot + 1 == sc.nb ? 0 : slot + 1; }
  return (uint32_t)k | (uint32_t)slot << 7;
}

// decode from (pos, st) until pos reaches `end` or the stream dies; returns the blocks completed on the way
DEC_HD uint32_t dec_run(const uint32_t *w, uint32_t nbits, uint32_t end, uint32_t &pos, uint32_t &st, const DecScan &sc, const DecTable *tabs)
{
  uint32_t n = 0;
  while (st != DEC_DEAD && pos < end) {
    int zz, val; bool done;
    const uint32_t ns = dec_step(w, nbits, pos, st, sc, tabs, zz, val, done);
    st = ns; n += done;
  }
  return n;
}

}  // namespace b200
