// decode_kernels.cu -- sm_90a kernels of the JPEG decompressor (see decode_kernels.cuh).
// Compile with: -gencode arch=compute_90a,code=sm_90a -fmad=false -lineinfo
#include "kernels.cuh"
#include "decode_kernels.cuh"

namespace b200 {

#include "zigzag.inc"

// ================================================================ Huffman decode (jpeg_read_coefficients)
// Speculative decode with self-synchronisation over DEC_SUB_BITS-bit subsequences of every restart segment of every
// first scan (sequential, DC first, AC first; decode.cuh).
// A subsequence's record holds the (position, state) its last decode started from and where it stopped.  Every
// segment's first subsequence starts exact; any other is right once its start equals its predecessor's stop.

// the segment holding global subsequence j (segments are ordered by sub0)
__device__ __forceinline__ int dec_find_seg(const DecSeg *__restrict__ segs, int nsegs, long long j)
{
  int lo = 0, hi = nsegs - 1;
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (segs[mid].sub0 <= j) lo = mid; else hi = mid - 1; }
  return lo;
}

// one CTA = DEC_CTA consecutive subsequences: decode each from a guessed start (the block's DC, slot 0), then
// re-decode every subsequence whose start differs from its predecessor's stop until none does (at most DEC_CTA rounds)
__global__ void __launch_bounds__(DEC_CTA) k_dec_sync(const uint32_t *__restrict__ words, const DecSeg *__restrict__ segs, int nsegs,
                                                      const DecScan *__restrict__ scans, const DecTable *__restrict__ tabs,
                                                      DecRec *__restrict__ rec, long long nsub, int *__restrict__ max_rounds)
{
  __shared__ uint32_t s_pos[DEC_CTA], s_st[DEC_CTA];
  const int t = threadIdx.x;
  const long long j = (long long)blockIdx.x * DEC_CTA + t;
  const bool live = j < nsub;
  DecSeg g; g.nbits = 0; g.scan = 0; const uint32_t *w = words; uint32_t a = 0, b = 0;
  bool seg_first = true;
  uint32_t in_pos = 0, in_st = 0, pos = 0, st = 0, cnt = 0;
  if (live) {
    g = segs[dec_find_seg(segs, nsegs, j)];
    w = words + g.word0;
    a = (uint32_t)(j - g.sub0) * DEC_SUB_BITS; b = min(a + DEC_SUB_BITS, g.nbits);
    seg_first = j == g.sub0;
    in_pos = pos = a; in_st = st = 0;
    cnt = dec_run(w, g.nbits, b, pos, st, scans[g.scan], tabs);
  }
  s_pos[t] = pos; s_st[t] = st;
  int rounds = 0;
  for (;;) {
    __syncthreads();
    const bool has_pred = live && !seg_first && t > 0;
    const uint32_t pp = has_pred ? s_pos[t - 1] : 0, ps = has_pred ? s_st[t - 1] : 0;
    __syncthreads();
    const bool change = has_pred && (pp != in_pos || ps != in_st);
    if (change) {
      in_pos = pos = pp; in_st = st = ps;
      cnt = dec_run(w, g.nbits, b, pos, st, scans[g.scan], tabs);
      s_pos[t] = pos; s_st[t] = st;
    }
    if (!__syncthreads_or(change)) break;
    rounds++;
  }
  if (live) { DecRec r; r.in_pos = in_pos; r.in_st = in_st; r.out_pos = pos; r.out_st = st; r.count = cnt; r.pad = 0; rec[j] = r; }
  if (t == 0 && rounds) atomicMax(max_rounds, rounds);
}

// one thread per segment: the subsequences that open a CTA inside the segment started from a guess; decode them
// again from their predecessor's stop until one agrees with what it recorded (the rest of its CTA then holds)
__global__ void __launch_bounds__(128) k_dec_fix(const uint32_t *__restrict__ words, const DecSeg *__restrict__ segs, int nsegs,
                                                 const DecScan *__restrict__ scans, const DecTable *__restrict__ tabs,
                                                 DecRec *__restrict__ rec, unsigned long long *__restrict__ redone)
{
  const int si = blockIdx.x * blockDim.x + threadIdx.x;
  if (si >= nsegs) return;
  const DecSeg g = segs[si];
  if (g.nsub == 1) return;
  const DecScan &sc = scans[g.scan];
  const uint32_t *w = words + g.word0;
  const long long end = g.sub0 + g.nsub;
  unsigned long long n = 0;
  for (long long j = (g.sub0 / DEC_CTA + 1) * DEC_CTA; j < end; j += DEC_CTA) {
    long long q = j;
    for (; q < end; q++) {
      const DecRec p = rec[q - 1];
      DecRec r = rec[q];
      if (r.in_pos == p.out_pos && r.in_st == p.out_st) break;
      const uint32_t a = (uint32_t)(q - g.sub0) * DEC_SUB_BITS, b = min(a + DEC_SUB_BITS, g.nbits);
      r.in_pos = p.out_pos; r.in_st = p.out_st;
      uint32_t pos = r.in_pos, st = r.in_st;
      r.count = dec_run(w, g.nbits, b, pos, st, sc, tabs);
      r.out_pos = pos; r.out_st = st;
      rec[q] = r; n++;
    }
  }
  if (n) atomicAdd(redone, n);
}

// exclusive scan of the blocks completed per subsequence: in tiles of 1024 (pre), then over the tile sums (tsum)
__global__ void __launch_bounds__(1024) k_dec_scan_tiles(const DecRec *__restrict__ rec, long long nsub, uint32_t *__restrict__ pre, unsigned long long *__restrict__ tsum)
{
  __shared__ uint32_t s_w[32];
  const long long j = (long long)blockIdx.x * 1024 + threadIdx.x;
  const uint32_t v = j < nsub ? rec[j].count : 0u;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint32_t x = v;
  for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
  if (lane == 31) s_w[wid] = x;
  __syncthreads();
  if (wid == 0) {
    uint32_t y = s_w[lane];
    for (int o = 1; o < 32; o <<= 1) { const uint32_t z = __shfl_up_sync(0xffffffffu, y, o); if (lane >= o) y += z; }
    s_w[lane] = y;
  }
  __syncthreads();
  const uint32_t incl = x + (wid ? s_w[wid - 1] : 0u);
  if (j < nsub) pre[j] = incl - v;
  if (threadIdx.x == 1023) tsum[blockIdx.x] = incl;
}
__global__ void __launch_bounds__(1024) k_dec_scan_sums(unsigned long long *__restrict__ tsum, long long ntiles)
{
  __shared__ unsigned long long s_w[32];
  __shared__ unsigned long long s_carry;
  if (threadIdx.x == 0) s_carry = 0;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (long long base = 0; base < ntiles; base += 1024) {
    __syncthreads();
    const long long i = base + threadIdx.x;
    const unsigned long long v = i < ntiles ? tsum[i] : 0ull;
    unsigned long long x = v;
    for (int o = 1; o < 32; o <<= 1) { const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) s_w[wid] = x;
    __syncthreads();
    if (wid == 0) {
      unsigned long long y = s_w[lane];
      for (int o = 1; o < 32; o <<= 1) { const unsigned long long z = __shfl_up_sync(0xffffffffu, y, o); if (lane >= o) y += z; }
      s_w[lane] = y;
    }
    __syncthreads();
    const unsigned long long incl = x + (wid ? s_w[wid - 1] : 0ull) + s_carry;
    if (i < ntiles) tsum[i] = incl - v;
    __syncthreads();
    if (threadIdx.x == 1023) s_carry = incl;
  }
}

__device__ __forceinline__ unsigned long long dec_prefix(const uint32_t *pre, const unsigned long long *tsum, long long j)
{
  return tsum[j >> 10] + pre[j];
}

__device__ __forceinline__ int16_t *dec_block(const DecOut &o, const DecScan &sc, long long mcu, int slot)
{
  const int c = sc.comp[slot];
  const long long col = (mcu % sc.per_row) * sc.mx[c] + sc.dx[slot], row = (mcu / sc.per_row) * sc.my[c] + sc.dy[slot];
  if (col >= sc.wib[c] || row >= sc.hib[c]) return nullptr;        // a dummy block of an interleaved scan
  return o.plane[c] + (sc.base[c] + row * sc.wib[c] + col) * 64;
}

// the blocks subsequence j writes (k_dec_write), from (pos, st) to the first block start at or past bit b
template <bool PROG>
__device__ __forceinline__ void dec_write_blocks(const uint32_t *w, const DecSeg &g, const DecScan &sc, const DecTable *tabs, uint32_t pos, uint32_t st,
                                                 uint32_t b, long long blk, long long need, const DecOut &o, int *dcd, uint32_t *status)
{
  bool skip = (st & 127) != 0 && st != DEC_DEAD;         // the block in progress belongs to the predecessor
  int16_t *dst = nullptr;
  while (st != DEC_DEAD && blk < need) {
    if ((st & 127) == 0) {                                // a block starts here
      if (pos >= b) break;
      dst = dec_block(o, sc, g.mcu0 + blk / sc.nb, (int)(st >> 7));
    }
    int zz, val, done;
    st = dec_step<PROG>(w, g.nbits, pos, st, sc, tabs, zz, val, done);
    if (st == DEC_DEAD) break;
    if (!skip) {
      if (zz == 0) dcd[g.blk0 + blk] = val;
      else if (PROG && zz > sc.Se) atomicOr(&status[sc.img], 2u);
      else if (zz > 0 && dst) dst[c_zz[zz]] = PROG ? (int16_t)((unsigned)val << sc.Al) : (int16_t)val;
    }
    if (done) { blk += done; skip = false; }
  }
}

// one thread per subsequence: decode again from the synchronised start and write the AC coefficients of every block
// that starts inside the subsequence (finishing the last one past its end) into the planes (zeroed before), the DC
// differences into dcd; the segment's last subsequence checks that the segment holds all its MCUs.  AC first values
// are stored shifted by Al; one past a band that ends before 63 (it would land in another scan's band) sets status 2.
__global__ void __launch_bounds__(128) k_dec_write(const uint32_t *__restrict__ words, const DecSeg *__restrict__ segs, int nsegs,
                                                   const DecScan *__restrict__ scans, const DecTable *__restrict__ tabs,
                                                   const DecRec *__restrict__ rec, long long nsub, const uint32_t *__restrict__ pre,
                                                   const unsigned long long *__restrict__ tsum, const DecOut *__restrict__ o, int *__restrict__ dcd,
                                                   uint32_t *__restrict__ status)
{
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= nsub) return;
  const DecSeg g = segs[dec_find_seg(segs, nsegs, j)];
  const DecScan &sc = scans[g.scan];
  const uint32_t *w = words + g.word0;
  const DecRec r = rec[j];
  const long long need = (long long)g.nmcu * sc.nb;
  const unsigned long long seg_base = dec_prefix(pre, tsum, g.sub0);
  const long long blk = (long long)(dec_prefix(pre, tsum, j) - seg_base);
  if (j == g.sub0 + g.nsub - 1 && blk + (long long)r.count < need) atomicOr(&status[sc.img], 1u);
  const uint32_t b = min((uint32_t)(j - g.sub0 + 1) * DEC_SUB_BITS, g.nbits);
  if (sc.kind == DEC_SEQ) dec_write_blocks<false>(w, g, sc, tabs, r.in_pos, r.in_st, b, blk, need, *o, dcd, status);
  else dec_write_blocks<true>(w, g, sc, tabs, r.in_pos, r.in_st, b, blk, need, *o, dcd, status);
}

// one warp per (segment, scan component): DC values = running sum of the differences over the component's blocks in
// scan order, dummy blocks included, reset at the segment start (decode_mcu: int accumulation, JCOEF store of the
// sum shifted by Al)
__global__ void __launch_bounds__(128) k_dec_dc(const DecSeg *__restrict__ segs, int nsegs, const DecScan *__restrict__ scans,
                                                const int *__restrict__ dcd, const DecOut *__restrict__ o)
{
  const long long gw = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (gw >= (long long)nsegs * 4) return;
  const DecSeg g = segs[gw >> 2];
  const int k = (int)(gw & 3);
  const DecScan &sc = scans[g.scan];
  if (k >= sc.ncomp || sc.kind == DEC_AC_FIRST) return;
  const int cnt = sc.cnt[k], first = sc.first[k];
  const long long total = (long long)g.nmcu * cnt;
  unsigned carry = 0;
  for (long long base = 0; base < total; base += 32) {
    const long long e = base + lane;
    unsigned v = 0; long long m = 0; int slot = 0;
    if (e < total) { m = e / cnt; slot = first + (int)(e % cnt); v = (unsigned)dcd[g.blk0 + m * sc.nb + slot]; }
    unsigned x = v;
    for (int of = 1; of < 32; of <<= 1) { const unsigned y = __shfl_up_sync(0xffffffffu, x, of); if (lane >= of) x += y; }
    const unsigned s = x + carry;
    if (e < total) { int16_t *dst = dec_block(*o, sc, g.mcu0 + m, slot); if (dst) dst[0] = (int16_t)(s << sc.Al); }
    carry = __shfl_sync(0xffffffffu, s, 31);
  }
}

// ---------------------------------------------------------------- successive-approximation refinement scans

// one thread per block of every DC refinement segment (decode_mcu_DC_refine, jdphuff.c:443-489): block j of a segment
// ORs bit j of the segment, at 1 << Al, into its DC.  Refinements of different Al touch different bits, so every DC
// refinement scan runs in this one launch; the OR goes through the 32-bit word holding coefficients 0 and 1.  A
// segment with fewer bits than blocks sets status 1.
__global__ void __launch_bounds__(128) k_dec_dc_refine(const uint32_t *__restrict__ words, const DecSeg *__restrict__ segs, int nsegs,
                                                       const DecScan *__restrict__ scans, long long nblocks, const DecOut *__restrict__ o,
                                                       uint32_t *__restrict__ status)
{
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= nblocks) return;
  int lo = 0, hi = nsegs - 1;
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (segs[mid].blk0 <= j) lo = mid; else hi = mid - 1; }
  const DecSeg g = segs[lo];
  const DecScan &sc = scans[g.scan];
  const long long b = j - g.blk0;
  if (b >= (long long)g.nbits) { if (b == (long long)g.nbits) atomicOr(&status[sc.img], 1u); return; }
  if (!((dec_bswap(words[g.word0 + (b >> 5)]) >> (31 - (b & 31))) & 1u)) return;
  int16_t *dst = dec_block(*o, sc, g.mcu0 + b / sc.nb, (int)(b % sc.nb));
  if (dst) atomicOr(reinterpret_cast<unsigned *>(dst), (1u << sc.Al) & 0xFFFFu);
}

// the zigzag index of each natural position (the inverse of c_zz)
__constant__ uint8_t c_unzz[64] = {
   0,  1,  5,  6, 14, 15, 27, 28,  2,  4,  7, 13, 16, 26, 29, 42,  3,  8, 12, 17, 25, 30, 41, 43,  9, 11, 18, 24, 31, 40, 44, 53,
  10, 19, 23, 32, 39, 45, 52, 54, 20, 22, 33, 38, 46, 51, 55, 60, 21, 34, 37, 47, 50, 56, 59, 61, 35, 36, 48, 49, 57, 58, 62, 63};

// n (<= 64) bits at pos, MSB first, into the low bits
__device__ __forceinline__ unsigned long long dec_bits(const uint32_t *w, uint32_t pos, int n)
{
  unsigned long long x = 0;
  while (n > 0) { const int c = n < 24 ? n : 24; x = (x << c) | (dec_window(w, pos) >> (32 - c)); pos += c; n -= c; }
  return x;
}

// bits (MSB first: the first bit for the lowest set bit of mask) spread over the set bits of mask
__device__ __forceinline__ unsigned long long dec_deposit(unsigned long long mask, unsigned long long bits, int n)
{
  unsigned long long r = 0;
  for (int i = n - 1; i >= 0; i--) { const unsigned long long lowest = mask & (0ull - mask); if ((bits >> i) & 1ull) r |= lowest; mask ^= lowest; }
  return r;
}

// One warp per AC refinement segment of one level (decode_mcu_AC_refine, jdphuff.c:497-640), its blocks in order: the
// bits a block takes depend on which coefficients of its band are already nonzero, so a segment is decoded serially.
// Each block's 128 bytes come in one coalesced load (the next block's is in flight meanwhile); a ballot gives the
// band's nonzero mask in zigzag order; every lane runs the same symbol decode, walking the correction bits over the
// mask's set bits; the lanes then write the changed coefficients back.  Status: 1 for an invalid code or too few bits,
// 2 for a new coefficient past a band that ends before 63, 4 for a symbol of size other than 1.
__global__ void __launch_bounds__(128) k_dec_ac_refine(const uint32_t *__restrict__ words, const DecSeg *__restrict__ segs, int nsegs,
                                                       const DecScan *__restrict__ scans, const DecTable *__restrict__ tabs,
                                                       const DecOut *__restrict__ o, uint32_t *__restrict__ status)
{
  const int gw = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (gw >= nsegs) return;
  const DecSeg g = segs[gw];
  const DecScan &sc = scans[g.scan];
  const DecTable &t = tabs[sc.tac[0]];
  const uint32_t *w = words + g.word0;
  const int Ss = sc.Ss, Se = sc.Se, p1 = 1 << sc.Al, m1 = -p1;
  const unsigned long long band = (Se == 63 ? ~0ull : (1ull << (Se + 1)) - 1) & ~((1ull << Ss) - 1);
  const int z0 = c_unzz[2 * lane], z1 = c_unzz[2 * lane + 1], n0 = c_zz[lane], n1 = c_zz[lane + 32];
  const long long need = g.nmcu;
  uint32_t pos = 0, eobrun = 0, err = 0;
  unsigned *blk = need ? reinterpret_cast<unsigned *>(dec_block(*o, sc, g.mcu0, 0)) : nullptr;
  unsigned nxt = blk ? blk[lane] : 0u;
  for (long long b = 0; b < need && !err; b++) {
    unsigned *cur = blk;
    const unsigned word = nxt;
    if (b + 1 < need) { blk = reinterpret_cast<unsigned *>(dec_block(*o, sc, g.mcu0 + b + 1, 0)); nxt = blk[lane]; }
    const int16_t c0 = (int16_t)(word & 0xFFFFu), c1 = (int16_t)(word >> 16);
    // the nonzero coefficients of the band as a zigzag mask: lane l looks up zigzag indices l and l + 32
    const unsigned q0 = __shfl_sync(0xffffffffu, word, n0 >> 1), q1 = __shfl_sync(0xffffffffu, word, n1 >> 1);
    const unsigned long long zmask = ((unsigned long long)__ballot_sync(0xffffffffu, ((n0 & 1) ? q0 >> 16 : q0 & 0xFFFFu) != 0) |
                                      (unsigned long long)__ballot_sync(0xffffffffu, ((n1 & 1) ? q1 >> 16 : q1 & 0xFFFFu) != 0) << 32) & band;
    unsigned long long inc = 0, newnz = 0, newneg = 0;
    int k = Ss;
    if (eobrun == 0) {
      for (; k <= Se; k++) {
        int sym;
        const uint32_t win = dec_window(w, pos);
        const int len = dec_symbol(win, t, sym);
        if (!len || pos + (uint32_t)len > g.nbits) { err = 1; break; }
        pos += len;
        int r = sym >> 4, s = sym & 15;
        bool neg = false;
        if (s) {
          if (s != 1) { err = 4; break; }
          if (pos + 1 > g.nbits) { err = 1; break; }
          neg = !((dec_window(w, pos) >> 31) & 1u); pos++;
        } else if (r != 15) {
          if (pos + (uint32_t)r > g.nbits) { err = 1; break; }
          eobrun = (1u << r) + (r ? (uint32_t)dec_bits(w, pos, r) : 0u); pos += r;
          break;
        }
        // the (r + 1)-th zero at or after k is the target; the nonzero ones before it take a correction bit each
        unsigned long long zeros = ~zmask & band & ~((1ull << k) - 1);
        for (int i = 0; i < r && zeros; i++) zeros &= zeros - 1;
        const int target = zeros ? __ffsll((long long)zeros) - 1 : Se + 1;
        const unsigned long long before = zmask & ~((1ull << k) - 1) & (target >= 64 ? ~0ull : (1ull << target) - 1);
        const int nc = __popcll(before);
        if (pos + (uint32_t)nc > g.nbits) { err = 1; break; }
        inc |= dec_deposit(before, dec_bits(w, pos, nc), nc); pos += nc;
        k = target;
        if (s) {
          if (k > Se && Se < 63) { err = 2; break; }
          const int z = k > 63 ? 63 : k;
          newnz |= 1ull << z; if (neg) newneg |= 1ull << z; else newneg &= ~(1ull << z);
        }
      }
    }
    if (!err && eobrun > 0) {
      const unsigned long long rest = zmask & (k >= 64 ? 0ull : ~((1ull << k) - 1));
      const int nc = __popcll(rest);
      if (pos + (uint32_t)nc > g.nbits) err = 1;
      else { inc |= dec_deposit(rest, dec_bits(w, pos, nc), nc); pos += nc; eobrun--; }
    }
    if (err || !(inc | newnz)) continue;
    int v0 = c0, v1 = c1;
    if ((newnz >> z0) & 1) v0 = ((newneg >> z0) & 1) ? m1 : p1;
    else if (((inc >> z0) & 1) && !(v0 & p1)) v0 += v0 >= 0 ? p1 : m1;
    if ((newnz >> z1) & 1) v1 = ((newneg >> z1) & 1) ? m1 : p1;
    else if (((inc >> z1) & 1) && !(v1 & p1)) v1 += v1 >= 0 ? p1 : m1;
    cur[lane] = (unsigned)(uint16_t)v0 | (unsigned)(uint16_t)v1 << 16;
  }
  if (err && lane == 0) atomicOr(&status[sc.img], (uint32_t)err);
}

void launch_decode_refine(const uint32_t *words, const DecSeg *dcr, int ndcr, long long dcr_blocks, const DecSeg *acr, const int *acr_level, int nlevels,
                          const DecScan *scans, const DecTable *tabs, const DecOut *o, uint32_t *status, cudaEvent_t *marks, cudaStream_t s)
{
  if (ndcr) { k_dec_dc_refine<<<(unsigned)((dcr_blocks + 127) / 128), 128, 0, s>>>(words, dcr, ndcr, scans, dcr_blocks, o, status); LAUNCHED(); }
  cudaEventRecord(marks[0], s);
  for (int l = 0; l < nlevels; l++) {
    const int n = acr_level[l + 1] - acr_level[l];
    if (n) { k_dec_ac_refine<<<(unsigned)((n * 32 + 127) / 128), 128, 0, s>>>(words, acr + acr_level[l], n, scans, tabs, o, status); LAUNCHED(); }
  }
  cudaEventRecord(marks[1], s);
}

void launch_decode(const uint32_t *words, const DecSeg *segs, int nsegs, const DecScan *scans, const DecTable *tabs, long long nsub,
                   DecRec *rec, uint32_t *pre, unsigned long long *tsum, int *dcd, const DecOut *o, uint32_t *status,
                   int *max_rounds, unsigned long long *redone, cudaEvent_t *marks, cudaStream_t s)
{
  const unsigned nb_sync = (unsigned)((nsub + DEC_CTA - 1) / DEC_CTA);
  const long long ntiles = (nsub + 1023) / 1024;
  cudaEventRecord(marks[0], s);
  k_dec_sync<<<nb_sync, DEC_CTA, 0, s>>>(words, segs, nsegs, scans, tabs, rec, nsub, max_rounds); LAUNCHED();
  cudaEventRecord(marks[1], s);
  k_dec_fix<<<(nsegs + 127) / 128, 128, 0, s>>>(words, segs, nsegs, scans, tabs, rec, redone); LAUNCHED();
  cudaEventRecord(marks[2], s);
  k_dec_scan_tiles<<<(unsigned)ntiles, 1024, 0, s>>>(rec, nsub, pre, tsum); LAUNCHED();
  k_dec_scan_sums<<<1, 1024, 0, s>>>(tsum, ntiles); LAUNCHED();
  cudaEventRecord(marks[3], s);
  k_dec_write<<<(unsigned)((nsub + 127) / 128), 128, 0, s>>>(words, segs, nsegs, scans, tabs, rec, nsub, pre, tsum, o, dcd, status); LAUNCHED();
  cudaEventRecord(marks[4], s);
  k_dec_dc<<<(unsigned)(((long long)nsegs * 4 * 32 + 127) / 128), 128, 0, s>>>(segs, nsegs, scans, dcd, o); LAUNCHED();
  cudaEventRecord(marks[5], s);
}

// ------------------------------------------------------------------ decompression to pixels: the stages behind the
// entropy decode of a default decompress object (JDCT_ISLOW, fancy upsampling, out_color_space of
// default_decompress_parms), sample for sample

// IDCT_range_limit (jdmaster.c prepare_range_limit_table) indexed with x & RANGE_MASK (jidctint.c:283-291): the low ten
// bits of x taken as a signed number, plus the level shift, clamped
__device__ __forceinline__ int idct_range_limit(int x)
{
  const int s = (((x & 1023) ^ 512) - 512) + 128;
  return min(max(s, 0), 255);
}

#define IDCT_BLOCKS 32           // blocks per CTA of k_idct_islow (8 lanes each)
#define IDCT_WS 73               // ints per block of its workspace: 8 rows of 9, and one more so that blocks start in different banks

// Where block lb of this CTA of an IDCT kernel lies, for output blocks of N x N samples: its index in the coefficient
// plane, its table's offset, the byte offset of its first sample row and the row pitch.  One-geometry form (RAGGED
// false): the plane holds [n][hib][wib] blocks, image i's table at i * qstride, the samples [n][hib * N][wib * N].
// Ragged form: work[blockIdx.x] names the image (imgs[]) the CTA works on; each image's blocks are padded to whole
// CTAs of BPC blocks, so a CTA never spans two images.
// PLANE form (one geometry): the samples go to pd's plane, image i's at i * pd.stride, rows pd.pitch apart; x0 / y0:
// the block's first column and row there, for the clipping to pd.cw x pd.ch.
struct IdctAt { bool valid; long long blk, q, o, pitch; int x0, y0; };
template <bool RAGGED, int BPC, int N, bool PLANE = false>
__device__ __forceinline__ IdctAt idct_at(int lb, int wib, int hib, long long nblocks, int qstride, const uint32_t *__restrict__ work,
                                          const IdctImg *__restrict__ imgs, const IdctDst &pd = IdctDst())
{
  IdctAt a;
  if (!RAGGED) {
    a.blk = (long long)blockIdx.x * BPC + lb;
    a.valid = a.blk < nblocks;
    const long long per = (long long)wib * hib, img = a.valid ? a.blk / per : 0, rem = a.blk - img * per;
    const int by = (int)(rem / wib), bx = (int)(rem - (long long)by * wib);
    a.q = img * qstride; a.pitch = (long long)wib * N;
    a.o = ((img * hib + by) * N) * a.pitch + bx * N;
    if (PLANE) { a.pitch = pd.pitch; a.o = img * pd.stride + (long long)by * N * pd.pitch + bx * N; a.x0 = bx * N; a.y0 = by * N; }
  } else {
    const IdctImg d = imgs[work[blockIdx.x]];
    const long long b = (long long)(blockIdx.x - d.cta0) * BPC + lb;
    a.valid = b < (long long)d.wib * d.hib;
    const int by = (int)(b / d.wib), bx = (int)(b - (long long)by * d.wib);
    a.blk = d.coef + b; a.q = d.tab; a.pitch = (long long)d.wib * N;
    a.o = d.out + (long long)by * N * a.pitch + bx * N;
  }
  return a;
}

// the PLANE store of one sample row of a block: its N samples, packed little-endian in lo and hi, clipped to the first n
// (none for n <= 0); whole aligned rows as one store
template <int N>
__device__ __forceinline__ void store_row_clipped(uint8_t *dst, unsigned lo, unsigned hi, int n)
{
  if (n >= N && (reinterpret_cast<uintptr_t>(dst) & (N - 1)) == 0) {
    if (N == 8) *reinterpret_cast<uint2 *>(dst) = make_uint2(lo, hi);
    else if (N == 4) *reinterpret_cast<uint32_t *>(dst) = lo;
    else if (N == 2) *reinterpret_cast<uint16_t *>(dst) = (uint16_t)lo;
    else *dst = (uint8_t)lo;
    return;
  }
#pragma unroll
  for (int k = 0; k < N; k++)
    if (k < n) dst[k] = (uint8_t)((k < 4 ? lo : hi) >> (8 * (k & 3)));
}

// jpeg_idct_islow (jidctint.c:171-419, 8-bit: CONST_BITS 13, PASS1_BITS 2) with the dequantization of jddctmgr.c:
// 134-146 (ISLOW_MULT_TYPE is a short: the table entries are taken as int16).  Eight lanes per block: each loads one
// 16-byte row of the JBLOCK, transforms one column into the int workspace (pass 1), then one row into eight samples
// (pass 2) stored as one 8-byte word.  The reference's shortcuts for all-zero columns and rows give what the general
// butterfly gives, so there is no branch.  Pass 1 keeps the reference's 64-bit intermediates (JLONG): a file may carry
// 16-bit coefficients under a 16-bit table; pass 2 needs bits 18..27 of its sums only, which 32-bit arithmetic keeps.
// coef: [nblocks][64] natural order ([n][hib][wib] blocks); quant: image i's table at quant + i * qstride;
// out: [n][hib * 8][wib * 8] samples, or with PLANE pd's plane (idct_at).
template <bool RAGGED, bool PLANE = false>
__global__ void __launch_bounds__(IDCT_BLOCKS * 8) k_idct_islow(const int16_t *__restrict__ coef, const uint16_t *__restrict__ quant, int qstride,
                                                                uint8_t *__restrict__ out, int wib, int hib, long long nblocks,
                                                                const uint32_t *__restrict__ work, const IdctImg *__restrict__ imgs,
                                                                IdctDst pd = IdctDst())
{
  __shared__ int4 s_coef[IDCT_BLOCKS * 8];
  __shared__ int s_ws[IDCT_BLOCKS * IDCT_WS];
  const int lb = threadIdx.x >> 3, lane = threadIdx.x & 7;
  const IdctAt at = idct_at<RAGGED, IDCT_BLOCKS, 8, PLANE>(lb, wib, hib, nblocks, qstride, work, imgs, pd);
  const bool valid = at.valid;
  s_coef[threadIdx.x] = valid ? reinterpret_cast<const int4 *>(coef)[at.blk * 8 + lane] : make_int4(0, 0, 0, 0);
  __syncwarp();
  // pass 1: column `lane`
  {
    const int16_t *c = reinterpret_cast<const int16_t *>(s_coef + lb * 8) + lane;
    const uint16_t *q = quant + at.q + lane;
    long long d[8];
#pragma unroll
    for (int r = 0; r < 8; r++) d[r] = (long long)c[r * 8] * (int16_t)q[r * 8];
    long long z2 = d[2], z3 = d[6];
    long long z1 = (z2 + z3) * 4433;
    long long tmp2 = z1 + z3 * -15137, tmp3 = z1 + z2 * 6270;
    z2 = d[0]; z3 = d[4];
    long long tmp0 = (z2 + z3) * 8192, tmp1 = (z2 - z3) * 8192;
    const long long tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    tmp0 = d[7]; tmp1 = d[5]; tmp2 = d[3]; tmp3 = d[1];
    z1 = tmp0 + tmp3; z2 = tmp1 + tmp2; z3 = tmp0 + tmp2;
    long long z4 = tmp1 + tmp3;
    const long long z5 = (z3 + z4) * 9633;
    tmp0 *= 2446; tmp1 *= 16819; tmp2 *= 25172; tmp3 *= 12299;
    z1 *= -7373; z2 *= -20995; z3 *= -16069; z4 *= -3196;
    z3 += z5; z4 += z5;
    tmp0 += z1 + z3; tmp1 += z2 + z4; tmp2 += z2 + z3; tmp3 += z1 + z4;
    int *ws = s_ws + lb * IDCT_WS + lane;
    ws[0 * 9] = (int)((tmp10 + tmp3 + 1024) >> 11); ws[7 * 9] = (int)((tmp10 - tmp3 + 1024) >> 11);
    ws[1 * 9] = (int)((tmp11 + tmp2 + 1024) >> 11); ws[6 * 9] = (int)((tmp11 - tmp2 + 1024) >> 11);
    ws[2 * 9] = (int)((tmp12 + tmp1 + 1024) >> 11); ws[5 * 9] = (int)((tmp12 - tmp1 + 1024) >> 11);
    ws[3 * 9] = (int)((tmp13 + tmp0 + 1024) >> 11); ws[4 * 9] = (int)((tmp13 - tmp0 + 1024) >> 11);
  }
  __syncwarp();
  // pass 2: row `lane`, modulo 2^32
  {
    const int *ws = s_ws + lb * IDCT_WS + lane * 9;
    unsigned d[8];
#pragma unroll
    for (int k = 0; k < 8; k++) d[k] = (unsigned)ws[k];
    unsigned z2 = d[2], z3 = d[6];
    unsigned z1 = (z2 + z3) * 4433u;
    unsigned tmp2 = z1 - z3 * 15137u, tmp3 = z1 + z2 * 6270u;
    unsigned tmp0 = (d[0] + d[4]) << 13, tmp1 = (d[0] - d[4]) << 13;
    const unsigned tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    tmp0 = d[7]; tmp1 = d[5]; tmp2 = d[3]; tmp3 = d[1];
    z1 = tmp0 + tmp3; z2 = tmp1 + tmp2; z3 = tmp0 + tmp2;
    unsigned z4 = tmp1 + tmp3;
    const unsigned z5 = (z3 + z4) * 9633u;
    tmp0 *= 2446u; tmp1 *= 16819u; tmp2 *= 25172u; tmp3 *= 12299u;
    z1 *= 0u - 7373u; z2 *= 0u - 20995u; z3 *= 0u - 16069u; z4 *= 0u - 3196u;
    z3 += z5; z4 += z5;
    tmp0 += z1 + z3; tmp1 += z2 + z4; tmp2 += z2 + z3; tmp3 += z1 + z4;
    const unsigned rnd = 1u << 17;
    const unsigned o0 = idct_range_limit((int)((tmp10 + tmp3 + rnd) >> 18)), o7 = idct_range_limit((int)((tmp10 - tmp3 + rnd) >> 18));
    const unsigned o1 = idct_range_limit((int)((tmp11 + tmp2 + rnd) >> 18)), o6 = idct_range_limit((int)((tmp11 - tmp2 + rnd) >> 18));
    const unsigned o2 = idct_range_limit((int)((tmp12 + tmp1 + rnd) >> 18)), o5 = idct_range_limit((int)((tmp12 - tmp1 + rnd) >> 18));
    const unsigned o3 = idct_range_limit((int)((tmp13 + tmp0 + rnd) >> 18)), o4 = idct_range_limit((int)((tmp13 - tmp0 + rnd) >> 18));
    if (valid) {
      uint8_t *dst = out + at.o + lane * at.pitch;
      const unsigned lo = o0 | o1 << 8 | o2 << 16 | o3 << 24, hi = o4 | o5 << 8 | o6 << 16 | o7 << 24;
      if (!PLANE) *reinterpret_cast<uint2 *>(dst) = make_uint2(lo, hi);
      else if (at.y0 + lane < pd.ch) store_row_clipped<8>(dst, lo, hi, pd.cw - at.x0);
    }
  }
}

void launch_idct_islow(const int16_t *coef, const uint16_t *quant, int qstride, uint8_t *out, int wib, int hib, int n, cudaStream_t s)
{
  const long long nblocks = (long long)n * wib * hib;
  k_idct_islow<false><<<(unsigned)((nblocks + IDCT_BLOCKS - 1) / IDCT_BLOCKS), IDCT_BLOCKS * 8, 0, s>>>(coef, quant, qstride, out, wib, hib, nblocks, nullptr, nullptr); LAUNCHED();
}

// the sample of a chroma plane at (row, col), both clamped to the real downsampled samples: the row above the first is
// the first and the row below the last real one is that row again (jdmainct.c set_wraparound_pointers :240-266,
// set_bottom_pointers :269-297); a column clamped the same way turns the general filter step into the reference's
// first / last column cases (3 * a + a = 4 * a)
__device__ __forceinline__ int up_at(const uint8_t *__restrict__ p, int pitch, int dw, int dh, int r, int c)
{
  return __ldg(p + (long long)min(max(r, 0), dh - 1) * pitch + min(max(c, 0), dw - 1));
}

// output pixels x0 .. x0+3 of row y of one chroma plane (dw x dh real samples): the upsamplers jinit_upsampler picks
// with do_fancy_upsampling (jdsample.c:444-530).  fancy: downsampled_width > 2, below which the 2:1 horizontal cases
// fall back to replication (h2v1_upsample, h2v2_upsample), which has no vertical filter either.
template <int HX, int VX>
__device__ __forceinline__ void upsample4(const uint8_t *__restrict__ p, int pitch, int dw, int dh, int x0, int y, bool fancy, int v[4])
{
  if (HX == 1 && VX == 1) {                               // fullsize_upsample (:129-135)
    const uchar4 q = __ldg(reinterpret_cast<const uchar4 *>(p + (long long)y * pitch + x0));
    v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
  } else if (HX == 1) {                                   // h1v2_fancy_upsample (:316-352): 3/4 nearer row + 1/4 further, bias 1 / 2
    const int r = y >> 1, r1 = (y & 1) ? r + 1 : r - 1, bias = (y & 1) ? 2 : 1;
#pragma unroll
    for (int k = 0; k < 4; k++) v[k] = (3 * up_at(p, pitch, dw, dh, r, x0 + k) + up_at(p, pitch, dw, dh, r1, x0 + k) + bias) >> 2;
  } else {
    const int c0 = x0 >> 1, r = VX == 2 ? y >> 1 : y;
    if (!fancy) {                                         // h2v1_upsample / h2v2_upsample (:205-266)
      const int a = up_at(p, pitch, dw, dh, r, c0), b = up_at(p, pitch, dw, dh, r, c0 + 1);
      v[0] = v[1] = a; v[2] = v[3] = b;
    } else if (VX == 1) {                                 // h2v1_fancy_upsample (:276-306)
      const int l = up_at(p, pitch, dw, dh, r, c0 - 1), a = up_at(p, pitch, dw, dh, r, c0), b = up_at(p, pitch, dw, dh, r, c0 + 1), n = up_at(p, pitch, dw, dh, r, c0 + 2);
      v[0] = (3 * a + l + 1) >> 2; v[1] = (3 * a + b + 2) >> 2; v[2] = (3 * b + a + 1) >> 2; v[3] = (3 * b + n + 2) >> 2;
    } else {                                              // h2v2_fancy_upsample (:362-411): column sums 3 * nearer row + further row
      const int r1 = (y & 1) ? r + 1 : r - 1;
      int cs[4];
#pragma unroll
      for (int k = 0; k < 4; k++) cs[k] = 3 * up_at(p, pitch, dw, dh, r, c0 - 1 + k) + up_at(p, pitch, dw, dh, r1, c0 - 1 + k);
      v[0] = (3 * cs[1] + cs[0] + 8) >> 4; v[1] = (3 * cs[1] + cs[2] + 7) >> 4; v[2] = (3 * cs[2] + cs[1] + 8) >> 4; v[3] = (3 * cs[2] + cs[3] + 7) >> 4;
    }
  }
}

// Sample planes -> interleaved pixels, each written once: chroma upsampling (upsample4), then ycc_rgb_convert with the
// tables of build_ycc_rgb_table (jdcolor.c:210-252, SCALEBITS 16) computed in place, or the components as they are
// (grayscale_convert, null_convert / rgb_rgb_convert for an RGB-coded file).  One thread makes four pixels of a row:
// the luma word and the chroma samples around it come through L1 (neighbouring threads and rows share them), the
// pixels leave as 4-byte words where the destination allows (aligned: base, pitch and stride multiples of 4), bytes at
// a ragged right edge.  y0 / c1 / c2: image 0's planes, strides in bytes; dw x dh: the real chroma samples.
template <int HX, int VX, int NC>
__global__ void __launch_bounds__(256) k_upsample_color(const uint8_t *__restrict__ y0, const uint8_t *__restrict__ c1, const uint8_t *__restrict__ c2,
                                                        int ypitch, long long ystride, int cpitch, long long cstride, int dw, int dh, bool fancy, bool ycc,
                                                        uint8_t *__restrict__ pix, long long row_pitch, long long image_stride, int W, int H, bool aligned)
{
  const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4, y = blockIdx.y * blockDim.y + threadIdx.y, img = blockIdx.z;
  if (x0 >= W || y >= H) return;
  const uchar4 l = __ldg(reinterpret_cast<const uchar4 *>(y0 + img * ystride + (long long)y * ypitch + x0));
  const int lum[4] = {l.x, l.y, l.z, l.w};
  uint8_t *dst = pix + img * image_stride + y * row_pitch + (long long)x0 * NC;
  const int nx = min(4, W - x0);
  if (NC == 1) {
    if (aligned && nx == 4) *reinterpret_cast<uchar4 *>(dst) = l;
    else for (int k = 0; k < nx; k++) dst[k] = (uint8_t)lum[k];
    return;
  }
  int cb[4], cr[4];
  upsample4<HX, VX>(c1 + img * cstride, cpitch, dw, dh, x0, y, fancy, cb);
  upsample4<HX, VX>(c2 + img * cstride, cpitch, dw, dh, x0, y, fancy, cr);
  uint8_t o[12];
#pragma unroll
  for (int k = 0; k < 4; k++) {
    if (ycc) {
      const int u = cb[k] - 128, w = cr[k] - 128;
      o[3 * k + 0] = (uint8_t)min(max(lum[k] + ((91881 * w + 32768) >> 16), 0), 255);
      o[3 * k + 1] = (uint8_t)min(max(lum[k] + ((-22554 * u + 32768 - 46802 * w) >> 16), 0), 255);
      o[3 * k + 2] = (uint8_t)min(max(lum[k] + ((116130 * u + 32768) >> 16), 0), 255);
    } else { o[3 * k + 0] = (uint8_t)lum[k]; o[3 * k + 1] = (uint8_t)cb[k]; o[3 * k + 2] = (uint8_t)cr[k]; }
  }
  if (aligned && nx == 4) {
#pragma unroll
    for (int k = 0; k < 3; k++) reinterpret_cast<uint32_t *>(dst)[k] = o[4 * k] | o[4 * k + 1] << 8 | o[4 * k + 2] << 16 | (uint32_t)o[4 * k + 3] << 24;
  } else {
#pragma unroll
    for (int k = 0; k < 12; k++) if (k < nx * 3) dst[k] = o[k];
  }
}

int launch_upsample_color(int hx, int vx, int nc, const uint8_t *const *planes, const int *pitch, const long long *stride, int dw, int dh, bool ycc,
                          uint8_t *pix, size_t row_pitch, size_t image_stride, int W, int H, int n, cudaStream_t s)
{
  const dim3 cta(64, 4), grid((unsigned)((W + 255) / 256), (unsigned)((H + 3) / 4), (unsigned)n);
  const bool aligned = reinterpret_cast<uintptr_t>(pix) % 4 == 0 && row_pitch % 4 == 0 && image_stride % 4 == 0;
  const bool fancy = dw > 2;
#define UPSAMPLE_CASE(HX, VX, NC) \
  if (hx == HX && vx == VX && nc == NC) { \
    k_upsample_color<HX, VX, NC><<<grid, cta, 0, s>>>(planes[0], planes[1], planes[2], pitch[0], stride[0], pitch[1], stride[1], dw, dh, fancy, ycc, \
                                                      pix, (long long)row_pitch, (long long)image_stride, W, H, aligned); LAUNCHED(); return 0; }
  UPSAMPLE_CASE(1, 1, 1) UPSAMPLE_CASE(1, 1, 3) UPSAMPLE_CASE(2, 1, 3) UPSAMPLE_CASE(1, 2, 3) UPSAMPLE_CASE(2, 2, 3)
#undef UPSAMPLE_CASE
  return -1;
}

// ------------------------------------------------------------------ decompression with the decompress object's options
// (scale_num / scale_denom, dct_method, do_fancy_upsampling, out_color_space): the reduced IDCTs of jidctred.c, the
// ifast and float IDCTs, and one upsampling / colour conversion kernel whose choices are parameters

// jpeg_idct_4x4 / jpeg_idct_2x2 (jidctred.c:121-275, 279-387; CONST_BITS 13, PASS1_BITS 2, JLONG intermediates) and
// jpeg_idct_1x1 (:390-407), with the islow-style table (ISLOW_MULT_TYPE int without SIMD: the entries as unsigned
// 16-bit values).  N = 4 and 2: eight lanes per block as in k_idct_islow; lane r loads row r, lane c transforms column c
// (column 4, and for N = 2 columns 2, 4 and 6, are skipped as the reference skips them), lanes 0 .. N-1 one row each.
// The reference's shortcuts for all-zero AC columns and rows give what the general path gives (pass 1: DESCALE of
// dq << (CONST_BITS + 1 or 2) is dq << PASS1_BITS, truncated to int the same way; pass 2: both are DESCALE(w0, 5)), so
// there is no branch.  N = 1: one thread per block reads the DC term only.
// out: [n][hib * N][wib * N] samples, or with PLANE pd's plane (idct_at).  T: the table entries' type, uint16_t, or int
// for the ifast multiplier table a TJSAMP_420 chroma component reads at 1/2 (products wrap modulo 2^32 as the
// reference's int arithmetic does).
template <int N, bool RAGGED, bool PLANE = false, typename T = uint16_t>
__global__ void __launch_bounds__(IDCT_BLOCKS * 8) k_idct_red(const int16_t *__restrict__ coef, const T *__restrict__ quant, int qstride,
                                                              uint8_t *__restrict__ out, int wib, int hib, long long nblocks,
                                                              const uint32_t *__restrict__ work, const IdctImg *__restrict__ imgs,
                                                              IdctDst pd = IdctDst())
{
  if (N == 1) {
    const IdctAt at = idct_at<RAGGED, 256, 1, PLANE>(threadIdx.x, wib, hib, nblocks, qstride, work, imgs, pd);
    if (!at.valid || (PLANE && (at.x0 >= pd.cw || at.y0 >= pd.ch))) return;
    const int dq = (int)__ldg(coef + at.blk * 64) * (int)__ldg(quant + at.q);
    out[at.o] = (uint8_t)idct_range_limit((int)(((long long)dq + 4) >> 3));
    return;
  }
  __shared__ int4 s_coef[IDCT_BLOCKS * 8];
  __shared__ int s_ws[IDCT_BLOCKS * IDCT_WS];
  const int lb = threadIdx.x >> 3, lane = threadIdx.x & 7;
  const IdctAt at = idct_at<RAGGED, IDCT_BLOCKS, N, PLANE>(lb, wib, hib, nblocks, qstride, work, imgs, pd);
  const bool valid = at.valid;
  s_coef[threadIdx.x] = valid ? reinterpret_cast<const int4 *>(coef)[at.blk * 8 + lane] : make_int4(0, 0, 0, 0);
  __syncwarp();
  const bool col_used = N == 4 ? lane != 4 : (lane & 1) || lane == 0;
  if (col_used) {                                         // pass 1: column `lane` -> ws rows 0 .. N-1
    const int16_t *c = reinterpret_cast<const int16_t *>(s_coef + lb * 8) + lane;
    const T *q = quant + at.q + lane;
    long long d[8];
#pragma unroll
    for (int r = 0; r < 8; r++) d[r] = (N == 4 && r == 4) || (N == 2 && (r == 2 || r == 4 || r == 6)) ? 0 : (long long)((int)c[r * 8] * (int)q[r * 8]);
    int *ws = s_ws + lb * IDCT_WS + lane;
    if (N == 4) {
      const long long t0 = d[0] * 16384, t2 = d[2] * 15137 + d[6] * -6270;
      const long long tmp10 = t0 + t2, tmp12 = t0 - t2;
      const long long o0 = d[7] * -1730 + d[5] * 11893 + d[3] * -17799 + d[1] * 8697;
      const long long o2 = d[7] * -4176 + d[5] * -4926 + d[3] * 7373 + d[1] * 20995;
      ws[0 * 9] = (int)((tmp10 + o2 + 2048) >> 12); ws[3 * 9] = (int)((tmp10 - o2 + 2048) >> 12);
      ws[1 * 9] = (int)((tmp12 + o0 + 2048) >> 12); ws[2 * 9] = (int)((tmp12 - o0 + 2048) >> 12);
    } else {
      const long long tmp10 = d[0] * 32768, o0 = d[7] * -5906 + d[5] * 6967 + d[3] * -10426 + d[1] * 29692;
      ws[0 * 9] = (int)((tmp10 + o0 + 4096) >> 13); ws[1 * 9] = (int)((tmp10 - o0 + 4096) >> 13);
    }
  }
  __syncwarp();
  if (valid && lane < N && (!PLANE || at.y0 + lane < pd.ch)) {   // pass 2: row `lane`
    const int *w = s_ws + lb * IDCT_WS + lane * 9;
    uint8_t *dst = out + at.o + lane * at.pitch;
    if (N == 4) {
      const long long t0 = (long long)w[0] * 16384, t2 = (long long)w[2] * 15137 + (long long)w[6] * -6270;
      const long long tmp10 = t0 + t2, tmp12 = t0 - t2;
      const long long z1 = w[7], z2 = w[5], z3 = w[3], z4 = w[1];
      const long long o0 = z1 * -1730 + z2 * 11893 + z3 * -17799 + z4 * 8697;
      const long long o2 = z1 * -4176 + z2 * -4926 + z3 * 7373 + z4 * 20995;
      const long long rnd = 1LL << 18;
      const unsigned s0 = idct_range_limit((int)((tmp10 + o2 + rnd) >> 19)), s3 = idct_range_limit((int)((tmp10 - o2 + rnd) >> 19));
      const unsigned s1 = idct_range_limit((int)((tmp12 + o0 + rnd) >> 19)), s2 = idct_range_limit((int)((tmp12 - o0 + rnd) >> 19));
      if (!PLANE) *reinterpret_cast<uint32_t *>(dst) = s0 | s1 << 8 | s2 << 16 | s3 << 24;
      else store_row_clipped<4>(dst, s0 | s1 << 8 | s2 << 16 | s3 << 24, 0, pd.cw - at.x0);
    } else {
      const long long tmp10 = (long long)w[0] * 32768;
      const long long o0 = (long long)w[7] * -5906 + (long long)w[5] * 6967 + (long long)w[3] * -10426 + (long long)w[1] * 29692;
      const long long rnd = 1LL << 19;
      const unsigned s0 = idct_range_limit((int)((tmp10 + o0 + rnd) >> 20)), s1 = idct_range_limit((int)((tmp10 - o0 + rnd) >> 20));
      if (!PLANE) *reinterpret_cast<uint16_t *>(dst) = (uint16_t)(s0 | s1 << 8);
      else store_row_clipped<2>(dst, s0 | s1 << 8, 0, pd.cw - at.x0);
    }
  }
}

#include "idct_scaled.inc"

// workspace ints per block of k_idct_scaled: rows of 9 (8 used), 8 rows below N = 8 else N, and one more so that
// blocks start in different banks
template <int N> __host__ __device__ constexpr int idct_scaled_ws() { return (N < 8 ? 8 : N) * 9 + 1; }

// jpeg_idct_3x3 .. jpeg_idct_16x16 but 4 and 8 (jidctint.c:427-2625; the passes as idct_scaled.inc folds them) with
// the islow-style table (entries taken as unsigned 16-bit values, as k_idct_red takes them).  Eight lanes per block:
// lane r loads coefficient row r; pass 1 runs lanes 0 .. M-1 over columns (M = N below 8, reading rows 0 .. N-1 only,
// else 8) into N workspace rows, in 64 bits as the reference's JLONG; pass 2 gives lane l rows l, l + 8 (N > 8), each
// from M workspace values, and stores its N samples byte by byte (rows of N samples at a pitch of wib * N bytes are
// not word-aligned for odd N).  out: [n][hib * N][wib * N] samples, or with PLANE pd's plane clipped to pd.cw x pd.ch.
template <int N, bool RAGGED, bool PLANE = false>
__global__ void __launch_bounds__(IDCT_BLOCKS * 8) k_idct_scaled(const int16_t *__restrict__ coef, const uint16_t *__restrict__ quant, int qstride,
                                                                 uint8_t *__restrict__ out, int wib, int hib, long long nblocks,
                                                                 const uint32_t *__restrict__ work, const IdctImg *__restrict__ imgs,
                                                                 IdctDst pd = IdctDst())
{
  constexpr int M = N < 8 ? N : 8, WS = idct_scaled_ws<N>();
  __shared__ int4 s_coef[IDCT_BLOCKS * 8];
  __shared__ int s_ws[IDCT_BLOCKS * WS];
  const int lb = threadIdx.x >> 3, lane = threadIdx.x & 7;
  const IdctAt at = idct_at<RAGGED, IDCT_BLOCKS, N, PLANE>(lb, wib, hib, nblocks, qstride, work, imgs, pd);
  const bool valid = at.valid;
  s_coef[threadIdx.x] = valid && lane < M ? reinterpret_cast<const int4 *>(coef)[at.blk * 8 + lane] : make_int4(0, 0, 0, 0);
  __syncwarp();
  if (lane < M) {                                          // pass 1: column `lane` -> ws rows 0 .. N-1
    const int16_t *c = reinterpret_cast<const int16_t *>(s_coef + lb * 8) + lane;
    const uint16_t *q = quant + at.q + lane;
    long long d[M];
#pragma unroll
    for (int r = 0; r < M; r++) d[r] = (long long)((int)c[r * 8] * (int)q[r * 8]);
    int o[N];
    idct_scaled_p1<N>(d, o);
    int *ws = s_ws + lb * WS + lane;
#pragma unroll
    for (int r = 0; r < N; r++) ws[r * 9] = o[r];
  }
  __syncwarp();
#pragma unroll
  for (int r0 = 0; r0 < N; r0 += 8) {                      // pass 2: row r0 + lane
    const int r = r0 + lane;
    if (!valid || r >= N || (PLANE && at.y0 + r >= pd.ch)) continue;
    const int *w = s_ws + lb * WS + r * 9;
    unsigned d[M], o[N];
#pragma unroll
    for (int k = 0; k < M; k++) d[k] = (unsigned)w[k];
    idct_scaled_p2<N>(d, o);
    uint8_t *dst = out + at.o + r * at.pitch;
    const int n = PLANE ? pd.cw - at.x0 : N;
#pragma unroll
    for (int x = 0; x < N; x++)
      if (x < n) dst[x] = (uint8_t)idct_range_limit((int)o[x]);
  }
}

// k_idct_scaled's instances, by N
template <bool RAGGED, bool PLANE>
static void launch_idct_scaled(int size, const int16_t *coef, const uint16_t *q, int qstride, uint8_t *out, int wib, int hib, long long nblocks,
                               unsigned grid, const uint32_t *work, const IdctImg *imgs, const IdctDst &d, cudaStream_t s)
{
  switch (size) {
#define IDCT_SCALED_CASE(NN) \
    case NN: k_idct_scaled<NN, RAGGED, PLANE><<<grid, IDCT_BLOCKS * 8, 0, s>>>(coef, q, qstride, out, wib, hib, nblocks, work, imgs, d); LAUNCHED(); break;
    IDCT_SCALED_CASE(3) IDCT_SCALED_CASE(5) IDCT_SCALED_CASE(6) IDCT_SCALED_CASE(7) IDCT_SCALED_CASE(9) IDCT_SCALED_CASE(10)
    IDCT_SCALED_CASE(11) IDCT_SCALED_CASE(12) IDCT_SCALED_CASE(13) IDCT_SCALED_CASE(14) IDCT_SCALED_CASE(15) IDCT_SCALED_CASE(16)
#undef IDCT_SCALED_CASE
    default: break;
  }
}

bool idct_size_scaled(int size) { return size >= 3 && size <= 16 && size != 4 && size != 8; }

// MULTIPLY of jidctfst.c (8-bit: CONST_BITS 8, no rounding): the int times a JLONG constant in 64 bits, shifted, and
// truncated back to DCTELEM (int)
__device__ __forceinline__ unsigned ifast_mul(unsigned v, int c)
{
  return (unsigned)(int)(((long long)(int)v * c) >> 8);
}

// one 8-point pass of jpeg_idct_ifast (jidctfst.c:171-368) on DCTELEM = int, modulo 2^32 as the reference's int
// arithmetic behaves where a 16-bit table makes it overflow; o[k] is output k of the pass
__device__ __forceinline__ void ifast_1d(const unsigned d[8], unsigned o[8])
{
  unsigned tmp10 = d[0] + d[4], tmp11 = d[0] - d[4];
  unsigned tmp13 = d[2] + d[6], tmp12 = ifast_mul(d[2] - d[6], 362) - tmp13;
  const unsigned tmp0 = tmp10 + tmp13, tmp3 = tmp10 - tmp13, tmp1 = tmp11 + tmp12, tmp2 = tmp11 - tmp12;
  const unsigned z13 = d[5] + d[3], z10 = d[5] - d[3], z11 = d[1] + d[7], z12 = d[1] - d[7];
  const unsigned tmp7 = z11 + z13;
  tmp11 = ifast_mul(z11 - z13, 362);
  const unsigned z5 = ifast_mul(z10 + z12, 473);
  tmp10 = ifast_mul(z12, 277) - z5;
  tmp12 = ifast_mul(z10, -669) + z5;
  const unsigned tmp6 = tmp12 - tmp7, tmp5 = tmp11 - tmp6, tmp4 = tmp10 + tmp5;
  o[0] = tmp0 + tmp7; o[7] = tmp0 - tmp7; o[1] = tmp1 + tmp6; o[6] = tmp1 - tmp6;
  o[2] = tmp2 + tmp5; o[5] = tmp2 - tmp5; o[4] = tmp3 + tmp4; o[3] = tmp3 - tmp4;
}

// jpeg_idct_ifast with its multiplier table (jddctmgr.c: quantval * aanscales descaled to IFAST_SCALE_BITS, int),
// image i's at mtab + i * qstride.  Shape of k_idct_islow.  The all-zero shortcuts give the general path's values.
template <bool RAGGED, bool PLANE = false>
__global__ void __launch_bounds__(IDCT_BLOCKS * 8) k_idct_ifast(const int16_t *__restrict__ coef, const int *__restrict__ mtab, int qstride,
                                                                uint8_t *__restrict__ out, int wib, int hib, long long nblocks,
                                                                const uint32_t *__restrict__ work, const IdctImg *__restrict__ imgs,
                                                                IdctDst pd = IdctDst())
{
  __shared__ int4 s_coef[IDCT_BLOCKS * 8];
  __shared__ int s_ws[IDCT_BLOCKS * IDCT_WS];
  const int lb = threadIdx.x >> 3, lane = threadIdx.x & 7;
  const IdctAt at = idct_at<RAGGED, IDCT_BLOCKS, 8, PLANE>(lb, wib, hib, nblocks, qstride, work, imgs, pd);
  const bool valid = at.valid;
  s_coef[threadIdx.x] = valid ? reinterpret_cast<const int4 *>(coef)[at.blk * 8 + lane] : make_int4(0, 0, 0, 0);
  __syncwarp();
  {
    const int16_t *c = reinterpret_cast<const int16_t *>(s_coef + lb * 8) + lane;
    const int *q = mtab + at.q + lane;
    unsigned d[8], o[8];
#pragma unroll
    for (int r = 0; r < 8; r++) d[r] = (unsigned)(int)c[r * 8] * (unsigned)__ldg(q + r * 8);
    ifast_1d(d, o);
    int *ws = s_ws + lb * IDCT_WS + lane;
#pragma unroll
    for (int r = 0; r < 8; r++) ws[r * 9] = (int)o[r];
  }
  __syncwarp();
  {
    const int *ws = s_ws + lb * IDCT_WS + lane * 9;
    unsigned d[8], o[8];
#pragma unroll
    for (int k = 0; k < 8; k++) d[k] = (unsigned)ws[k];
    ifast_1d(d, o);
    unsigned s[8];
#pragma unroll
    for (int k = 0; k < 8; k++) s[k] = idct_range_limit((int)o[k] >> 5);        // IDESCALE(x, PASS1_BITS + 3)
    if (valid) {
      uint8_t *dst = out + at.o + lane * at.pitch;
      const unsigned lo = s[0] | s[1] << 8 | s[2] << 16 | s[3] << 24, hi = s[4] | s[5] << 8 | s[6] << 16 | s[7] << 24;
      if (!PLANE) *reinterpret_cast<uint2 *>(dst) = make_uint2(lo, hi);
      else if (at.y0 + lane < pd.ch) store_row_clipped<8>(dst, lo, hi, pd.cw - at.x0);
    }
  }
}

// one 8-point pass of jpeg_idct_float (jidctflt.c:72-237) in the reference's operation order (the file is compiled
// with -fmad=false, so every product and sum is rounded on its own, as FAST_FLOAT float arithmetic is); z5: the
// centring term pass 2 adds to the DC input (0 in pass 1)
__device__ __forceinline__ void float_1d(const float d[8], float z5, float o[8])
{
  const float c1414 = (float)1.414213562, c1847 = (float)1.847759065, c1082 = (float)1.082392200, c2613 = (float)2.613125930;
  const float a = d[0] + z5;
  float tmp10 = a + d[4], tmp11 = a - d[4];
  float tmp13 = d[2] + d[6], tmp12 = (d[2] - d[6]) * c1414 - tmp13;
  const float tmp0 = tmp10 + tmp13, tmp3 = tmp10 - tmp13, tmp1 = tmp11 + tmp12, tmp2 = tmp11 - tmp12;
  const float z13 = d[5] + d[3], z10 = d[5] - d[3], z11 = d[1] + d[7], z12 = d[1] - d[7];
  const float tmp7 = z11 + z13;
  tmp11 = (z11 - z13) * c1414;
  const float zz = (z10 + z12) * c1847;
  tmp10 = zz - z12 * c1082;
  tmp12 = zz - z10 * c2613;
  const float tmp6 = tmp12 - tmp7, tmp5 = tmp11 - tmp6, tmp4 = tmp10 - tmp5;
  o[0] = tmp0 + tmp7; o[7] = tmp0 - tmp7; o[1] = tmp1 + tmp6; o[6] = tmp1 - tmp6;
  o[2] = tmp2 + tmp5; o[5] = tmp2 - tmp5; o[3] = tmp3 + tmp4; o[4] = tmp3 - tmp4;
}

// sample_range_limit[(int)x & RANGE_MASK] (jdmaster.c prepare_range_limit_table): 0 .. 255 as they are, 256 .. 639 are
// 255, 640 .. 1023 are 0.  (int) of a float beyond the int range is INT_MIN on x86 and saturates here; both land on 0.
__device__ __forceinline__ unsigned float_range_limit(float x)
{
  const int j = (int)x & 1023;
  return j < 256 ? j : j < 640 ? 255 : 0;
}

// jpeg_idct_float with its multiplier table (quantval * aanscalefactor[row] * aanscalefactor[col] in double, stored as
// float), image i's at mtab + i * qstride.  Shape of k_idct_islow.  The all-zero column shortcut gives the general
// path's values (x + 0 and x - 0 are x).
template <bool RAGGED>
__global__ void __launch_bounds__(IDCT_BLOCKS * 8) k_idct_float(const int16_t *__restrict__ coef, const float *__restrict__ mtab, int qstride,
                                                                uint8_t *__restrict__ out, int wib, int hib, long long nblocks,
                                                                const uint32_t *__restrict__ work, const IdctImg *__restrict__ imgs)
{
  __shared__ int4 s_coef[IDCT_BLOCKS * 8];
  __shared__ float s_ws[IDCT_BLOCKS * IDCT_WS];
  const int lb = threadIdx.x >> 3, lane = threadIdx.x & 7;
  const IdctAt at = idct_at<RAGGED, IDCT_BLOCKS, 8>(lb, wib, hib, nblocks, qstride, work, imgs);
  const bool valid = at.valid;
  s_coef[threadIdx.x] = valid ? reinterpret_cast<const int4 *>(coef)[at.blk * 8 + lane] : make_int4(0, 0, 0, 0);
  __syncwarp();
  {
    const int16_t *c = reinterpret_cast<const int16_t *>(s_coef + lb * 8) + lane;
    const float *q = mtab + at.q + lane;
    float d[8], o[8];
#pragma unroll
    for (int r = 0; r < 8; r++) d[r] = (float)c[r * 8] * (__ldg(q + r * 8) * 0.125f);
    float_1d(d, 0.f, o);
    float *ws = s_ws + lb * IDCT_WS + lane;
#pragma unroll
    for (int r = 0; r < 8; r++) ws[r * 9] = o[r];
  }
  __syncwarp();
  {
    const float *ws = s_ws + lb * IDCT_WS + lane * 9;
    float d[8], o[8];
#pragma unroll
    for (int k = 0; k < 8; k++) d[k] = ws[k];
    float_1d(d, 128.5f, o);
    unsigned s[8];
#pragma unroll
    for (int k = 0; k < 8; k++) s[k] = float_range_limit(o[k]);
    if (valid) {
      uint8_t *dst = out + at.o + lane * at.pitch;
      *reinterpret_cast<uint2 *>(dst) = make_uint2(s[0] | s[1] << 8 | s[2] << 16 | s[3] << 24, s[4] | s[5] << 8 | s[6] << 16 | s[7] << 24);
    }
  }
}

void launch_idct_opts(int size, int method, const int16_t *coef, const void *tab, int qstride, uint8_t *out, int wib, int hib, int n, cudaStream_t s)
{
  const long long nblocks = (long long)n * wib * hib;
  const unsigned grid8 = (unsigned)((nblocks + IDCT_BLOCKS - 1) / IDCT_BLOCKS);
  const uint16_t *q = static_cast<const uint16_t *>(tab);
  if (size == 1) { k_idct_red<1, false><<<(unsigned)((nblocks + 255) / 256), 256, 0, s>>>(coef, q, qstride, out, wib, hib, nblocks, nullptr, nullptr); LAUNCHED(); }
  else if (size == 2) { k_idct_red<2, false><<<grid8, IDCT_BLOCKS * 8, 0, s>>>(coef, q, qstride, out, wib, hib, nblocks, nullptr, nullptr); LAUNCHED(); }
  else if (size == 4) { k_idct_red<4, false><<<grid8, IDCT_BLOCKS * 8, 0, s>>>(coef, q, qstride, out, wib, hib, nblocks, nullptr, nullptr); LAUNCHED(); }
  else if (idct_size_scaled(size)) launch_idct_scaled<false, false>(size, coef, q, qstride, out, wib, hib, nblocks, grid8, nullptr, nullptr, IdctDst(), s);
  else if (method == 1) { k_idct_ifast<false><<<grid8, IDCT_BLOCKS * 8, 0, s>>>(coef, static_cast<const int *>(tab), qstride, out, wib, hib, nblocks, nullptr, nullptr); LAUNCHED(); }
  else if (method == 2) { k_idct_float<false><<<grid8, IDCT_BLOCKS * 8, 0, s>>>(coef, static_cast<const float *>(tab), qstride, out, wib, hib, nblocks, nullptr, nullptr); LAUNCHED(); }
  else launch_idct_islow(coef, q, qstride, out, wib, hib, n, s);
}

int idct_blocks_per_cta(int size) { return size == 1 ? 256 : IDCT_BLOCKS; }

void launch_idct_ragged(int size, int method, const int16_t *coef, const void *tab, uint8_t *out, const uint32_t *work, const IdctImg *imgs,
                        unsigned ncta, cudaStream_t s)
{
  const uint16_t *q = static_cast<const uint16_t *>(tab);
  if (size == 1) { k_idct_red<1, true><<<ncta, 256, 0, s>>>(coef, q, 0, out, 0, 0, 0, work, imgs); LAUNCHED(); }
  else if (size == 2) { k_idct_red<2, true><<<ncta, IDCT_BLOCKS * 8, 0, s>>>(coef, q, 0, out, 0, 0, 0, work, imgs); LAUNCHED(); }
  else if (size == 4) { k_idct_red<4, true><<<ncta, IDCT_BLOCKS * 8, 0, s>>>(coef, q, 0, out, 0, 0, 0, work, imgs); LAUNCHED(); }
  else if (idct_size_scaled(size)) launch_idct_scaled<true, false>(size, coef, q, 0, out, 0, 0, 0, ncta, work, imgs, IdctDst(), s);
  else if (method == 1) { k_idct_ifast<true><<<ncta, IDCT_BLOCKS * 8, 0, s>>>(coef, static_cast<const int *>(tab), 0, out, 0, 0, 0, work, imgs); LAUNCHED(); }
  else if (method == 2) { k_idct_float<true><<<ncta, IDCT_BLOCKS * 8, 0, s>>>(coef, static_cast<const float *>(tab), 0, out, 0, 0, 0, work, imgs); LAUNCHED(); }
  else { k_idct_islow<true><<<ncta, IDCT_BLOCKS * 8, 0, s>>>(coef, q, 0, out, 0, 0, 0, work, imgs); LAUNCHED(); }
}

// one output sample of a component plane (dw x dh real samples) at pixel (x, y): fullsize, replication by hr x vr
// (h2v1_upsample, h2v2_upsample, int_upsample and what the merged upsampler does to chroma, jdmerge.c), or the fancy
// filters of upsample4 evaluated for one pixel
__device__ __forceinline__ int up_one(const uint8_t *__restrict__ p, int pitch, int dw, int dh, int hr, int vr, bool fancy, int x, int y)
{
  if (hr == 1 && vr == 1) return __ldg(p + (long long)y * pitch + x);
  if (!fancy) return up_at(p, pitch, dw, dh, vr == 2 ? y >> 1 : y, hr == 2 ? x >> 1 : x);
  if (vr == 1) {                                          // h2v1_fancy_upsample
    const int c = x >> 1, a = up_at(p, pitch, dw, dh, y, c);
    return (x & 1) ? (3 * a + up_at(p, pitch, dw, dh, y, c + 1) + 2) >> 2 : (3 * a + up_at(p, pitch, dw, dh, y, c - 1) + 1) >> 2;
  }
  const int r = y >> 1, r1 = (y & 1) ? r + 1 : r - 1;
  if (hr == 1) return (3 * up_at(p, pitch, dw, dh, r, x) + up_at(p, pitch, dw, dh, r1, x) + ((y & 1) ? 2 : 1)) >> 2;   // h1v2_fancy_upsample
  const int c = x >> 1, cn = (x & 1) ? c + 1 : c - 1;     // h2v2_fancy_upsample
  const int s0 = 3 * up_at(p, pitch, dw, dh, r, c) + up_at(p, pitch, dw, dh, r1, c), s1 = 3 * up_at(p, pitch, dw, dh, r, cn) + up_at(p, pitch, dw, dh, r1, cn);
  return (3 * s0 + s1 + ((x & 1) ? 7 : 8)) >> 4;
}

// Sample planes -> pixels in the requested layout, one thread per pixel: each used component upsampled by up_one, then
// the deconverter jinit_color_deconverter picks (jdcolor.c:760-930, jdcolext.c): grayscale_convert, ycc_rgb_convert,
// null_convert / rgb_rgb_convert, gray_rgb_convert or rgb_gray_convert, into o.ps bytes with R, G, B at o.off[0..2]
// and 0xFF at o.off[3] where the pixel has a fourth byte.
__device__ __forceinline__ void upsample_pixel(const UpsOpt &o, long long img, uint8_t *__restrict__ row, int x, int y)
{
  int v[3] = {0, 0, 0};
#pragma unroll
  for (int c = 0; c < 3; c++)
    if (c < o.nin) v[c] = up_one(o.plane[c] + img * o.stride[c], o.pitch[c], o.dw[c], o.dh[c], o.hr[c], o.vr[c], o.fancy[c] != 0, x, y);
  uint8_t *d = row + (long long)x * o.ps;
  int r, g, b;
  switch (o.conv) {
  case UPS_GRAY: d[0] = (uint8_t)v[0]; return;
  case UPS_RGB_GRAY: d[0] = (uint8_t)((19595 * v[0] + 38470 * v[1] + 7471 * v[2] + 32768) >> 16); return;
  case UPS_YCC_RGB: {
    const int u = v[1] - 128, w = v[2] - 128;
    r = min(max(v[0] + ((91881 * w + 32768) >> 16), 0), 255);
    g = min(max(v[0] + ((-22554 * u + 32768 - 46802 * w) >> 16), 0), 255);
    b = min(max(v[0] + ((116130 * u + 32768) >> 16), 0), 255);
    break;
  }
  case UPS_GRAY_RGB: r = g = b = v[0]; break;
  default: r = v[0]; g = v[1]; b = v[2]; break;          // UPS_COPY3
  }
  d[o.off[0]] = (uint8_t)r; d[o.off[1]] = (uint8_t)g; d[o.off[2]] = (uint8_t)b;
  if (o.ps == 4) d[o.off[3]] = 0xFF;
}

// The 4-component form (UpsOpt4): the four components upsampled by up_one, then ycck_cmyk_convert (jdcolor.c:544-587:
// C, M and Y are 255 minus the R, G and B of ycc_rgb_convert, range-limited, and K passes through) or null_convert, into
// 4 bytes stored as one 32-bit word where the pixel's address is a multiple of 4.
__device__ __forceinline__ void upsample_pixel(const UpsOpt4 &o, long long img, uint8_t *__restrict__ row, int x, int y)
{
  int v[4];
#pragma unroll
  for (int c = 0; c < 4; c++) v[c] = up_one(o.plane[c] + img * o.stride[c], o.pitch[c], o.dw[c], o.dh[c], o.hr[c], o.vr[c], o.fancy[c] != 0, x, y);
  if (o.conv == UPS_YCCK_CMYK) {
    const int l = v[0], u = v[1] - 128, w = v[2] - 128;
    v[0] = 255 - min(max(l + ((91881 * w + 32768) >> 16), 0), 255);
    v[1] = 255 - min(max(l + ((-22554 * u + 32768 - 46802 * w) >> 16), 0), 255);
    v[2] = 255 - min(max(l + ((116130 * u + 32768) >> 16), 0), 255);
  }
  uint8_t *d = row + (long long)x * 4;
  if ((reinterpret_cast<uintptr_t>(d) & 3) == 0) *reinterpret_cast<uint32_t *>(d) = (uint32_t)v[0] | (uint32_t)v[1] << 8 | (uint32_t)v[2] << 16 | (uint32_t)v[3] << 24;
  else { d[0] = (uint8_t)v[0]; d[1] = (uint8_t)v[1]; d[2] = (uint8_t)v[2]; d[3] = (uint8_t)v[3]; }
}

// NC: 3 for UpsOpt (1- and 3-component files), 4 for UpsOpt4
template <int NC>
__global__ void __launch_bounds__(256) k_upsample_opts(UpsOptN<NC> o, uint8_t *__restrict__ pix, long long row_pitch, long long image_stride, int W, int H)
{
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y, img = blockIdx.z;
  if (x >= W || y >= H) return;
  upsample_pixel(o, img, pix + img * image_stride + (long long)y * row_pitch, x, y);
}

// k_upsample_opts over images of different geometry and conversion: work[blockIdx.x] names the image (imgs[]) whose
// 64 x 4 pixel tile the CTA makes, tile blockIdx.x - cta0 of its gx tiles a row; the image's sample planes are its own
// (UpsOpt::stride unused).  The descriptor is staged in shared memory once per CTA.
template <int NC>
__global__ void __launch_bounds__(256) k_upsample_ragged(const uint32_t *__restrict__ work, const UpsImgN<NC> *__restrict__ imgs)
{
  static_assert(sizeof(UpsImgN<NC>) % 4 == 0 && sizeof(UpsImgN<NC>) / 4 <= 256, "UpsImg is staged one word per thread");
  __shared__ UpsImgN<NC> d;
  const int tid = threadIdx.y * blockDim.x + threadIdx.x;
  if (tid < (int)(sizeof(UpsImgN<NC>) / 4)) reinterpret_cast<uint32_t *>(&d)[tid] = reinterpret_cast<const uint32_t *>(imgs + work[blockIdx.x])[tid];
  __syncthreads();
  const int t = (int)blockIdx.x - d.cta0, ty = t / d.gx;
  const int x = (t - ty * d.gx) * 64 + threadIdx.x, y = ty * 4 + threadIdx.y;
  if (x >= d.W || y >= d.H) return;
  upsample_pixel(d.o, 0, d.pix + (long long)y * d.row_pitch, x, y);
}

template <int NC>
void launch_upsample_opts(const UpsOptN<NC> &o, uint8_t *pix, size_t row_pitch, size_t image_stride, int W, int H, int n, cudaStream_t s)
{
  const dim3 cta(64, 4), grid((unsigned)((W + 63) / 64), (unsigned)((H + 3) / 4), (unsigned)n);
  k_upsample_opts<NC><<<grid, cta, 0, s>>>(o, pix, (long long)row_pitch, (long long)image_stride, W, H); LAUNCHED();
}
template void launch_upsample_opts<3>(const UpsOpt &, uint8_t *, size_t, size_t, int, int, int, cudaStream_t);
template void launch_upsample_opts<4>(const UpsOpt4 &, uint8_t *, size_t, size_t, int, int, int, cudaStream_t);

template <int NC>
void launch_upsample_ragged(const uint32_t *work, const UpsImgN<NC> *imgs, unsigned ncta, cudaStream_t s)
{
  k_upsample_ragged<NC><<<ncta, dim3(64, 4), 0, s>>>(work, imgs); LAUNCHED();
}
template void launch_upsample_ragged<3>(const uint32_t *, const UpsImg *, unsigned, cudaStream_t);
template void launch_upsample_ragged<4>(const uint32_t *, const UpsImg4 *, unsigned, cudaStream_t);

// tj3DecodeYUVPlanes8 with do_fancy_upsampling off: the merged upsampler (4:2:0, 4:2:2 to the RGB family) and
// int_upsample (4:4:0, 4:1:1, 4:4:1) both replicate chroma, so each pixel reads one luma and one sample of each chroma
// plane, then ycc_rgb_convert (jdcolor.c, SCALEBITS 16; the merged upsampler's tables give the same values),
// gray_rgb_convert or grayscale_convert.  One thread per pixel; rows past H are never made (rows_to_go).  It shares no
// code with k_upsample_opts, so that kernel and the pixel routes built on it stay as they are.
__global__ void __launch_bounds__(256) k_yuv_to_pixels(YuvPix d, uint8_t *__restrict__ pix, long long row_pitch, long long image_stride, int W, int H)
{
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  const long long img = blockIdx.z;
  if (x >= W || y >= H) return;
  const int l = __ldg(d.plane[0] + img * d.stride[0] + (long long)y * d.pitch[0] + x);
  uint8_t *o = pix + img * image_stride + (long long)y * row_pitch + (long long)x * d.ps;
  if (d.conv == UPS_GRAY) { o[0] = (uint8_t)l; return; }
  int r = l, g = l, b = l;
  if (d.conv == UPS_YCC_RGB) {
    const long long cy = y >> d.vs, cx = x >> d.hs;
    const int u = __ldg(d.plane[1] + img * d.stride[1] + cy * d.pitch[1] + cx) - 128;
    const int w = __ldg(d.plane[2] + img * d.stride[2] + cy * d.pitch[2] + cx) - 128;
    r = min(max(l + ((91881 * w + 32768) >> 16), 0), 255);
    g = min(max(l + ((-22554 * u + 32768 - 46802 * w) >> 16), 0), 255);
    b = min(max(l + ((116130 * u + 32768) >> 16), 0), 255);
  }
  o[d.off[0]] = (uint8_t)r; o[d.off[1]] = (uint8_t)g; o[d.off[2]] = (uint8_t)b;
  if (d.ps == 4) o[d.off[3]] = 0xFF;
}

void launch_yuv_to_pixels(const YuvPix &d, uint8_t *pix, size_t row_pitch, size_t image_stride, int W, int H, int n, cudaStream_t s)
{
  const dim3 cta(64, 4), grid((unsigned)((W + 63) / 64), (unsigned)((H + 3) / 4), (unsigned)n);
  k_yuv_to_pixels<<<grid, cta, 0, s>>>(d, pix, (long long)row_pitch, (long long)image_stride, W, H); LAUNCHED();
}

void launch_idct_plane(int size, int method, bool int_table, const int16_t *coef, const void *tab, int qstride, uint8_t *out, const IdctDst &d,
                       int wib, int hib, int n, cudaStream_t s)
{
  const long long nblocks = (long long)n * wib * hib;
  const unsigned grid8 = (unsigned)((nblocks + IDCT_BLOCKS - 1) / IDCT_BLOCKS);
  const uint16_t *q = static_cast<const uint16_t *>(tab);
  if (size == 1) { k_idct_red<1, false, true><<<(unsigned)((nblocks + 255) / 256), 256, 0, s>>>(coef, q, qstride, out, wib, hib, nblocks, nullptr, nullptr, d); LAUNCHED(); }
  else if (size == 2) { k_idct_red<2, false, true><<<grid8, IDCT_BLOCKS * 8, 0, s>>>(coef, q, qstride, out, wib, hib, nblocks, nullptr, nullptr, d); LAUNCHED(); }
  else if (size == 4 && int_table) { k_idct_red<4, false, true, int><<<grid8, IDCT_BLOCKS * 8, 0, s>>>(coef, static_cast<const int *>(tab), qstride, out, wib, hib, nblocks, nullptr, nullptr, d); LAUNCHED(); }
  else if (size == 4) { k_idct_red<4, false, true><<<grid8, IDCT_BLOCKS * 8, 0, s>>>(coef, q, qstride, out, wib, hib, nblocks, nullptr, nullptr, d); LAUNCHED(); }
  else if (idct_size_scaled(size)) launch_idct_scaled<false, true>(size, coef, q, qstride, out, wib, hib, nblocks, grid8, nullptr, nullptr, d, s);
  else if (method == 1) { k_idct_ifast<false, true><<<grid8, IDCT_BLOCKS * 8, 0, s>>>(coef, static_cast<const int *>(tab), qstride, out, wib, hib, nblocks, nullptr, nullptr, d); LAUNCHED(); }
  else { k_idct_islow<false, true><<<grid8, IDCT_BLOCKS * 8, 0, s>>>(coef, q, qstride, out, wib, hib, nblocks, nullptr, nullptr, d); LAUNCHED(); }
}

}  // namespace b200
