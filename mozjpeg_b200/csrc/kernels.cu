// kernels.cu -- sm_90a kernels of the JPEG-encode hot path (see kernels.cuh).
// Compile with: -gencode arch=compute_90a,code=sm_90a -fmad=false -lineinfo
#include "kernels.cuh"
#include <cuda_fp16.h>
#include <cuda.h>           // CUtensorMap (the encode function itself is fetched through the runtime, no libcuda link)
#include <cstdio>
#include <cstdlib>
#include <type_traits>

namespace b200 {

unsigned long long g_kernel_launches = 0;
#define LAUNCHED() (++g_kernel_launches)

// zigzag index -> natural index (jutils.c:59-70) and its inverse
__constant__ uint8_t c_zz[64] = {
   0,  1,  8, 16,  9,  2,  3, 10, 17, 24, 32, 25, 18, 11,  4,  5,
  12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,  6,  7, 14, 21, 28,
  35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
  58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
// natural index -> zigzag position
__constant__ uint8_t c_izz[64] = {
   0,  1,  5,  6, 14, 15, 27, 28,  2,  4,  7, 13, 16, 26, 29, 42,
   3,  8, 12, 17, 25, 30, 41, 43,  9, 11, 18, 24, 31, 40, 44, 53,
  10, 19, 23, 32, 39, 45, 52, 54, 20, 22, 33, 38, 46, 51, 55, 60,
  21, 34, 37, 47, 50, 56, 59, 61, 35, 36, 48, 49, 57, 58, 62, 63};
// the same table by column: byte r of c_izz_col[j] = zigzag position of natural index 8r + j (one 8-byte load per lane
// instead of eight byte loads at lane-dependent constant addresses, which the constant cache serialises)
__constant__ unsigned long long c_izz_col[8] = {0x2315140a09030200ull, 0x242216130b080401ull, 0x30252117120c0705ull, 0x312f262018110d06ull, 0x39322e271f19100eull, 0x3a38332d281e1a0full, 0x3e3b37342c291d1bull, 0x3f3d3c36352b2a1cull};
#ifndef FWD_KZ_PACKED
#define FWD_KZ_PACKED 1
#endif
#define ZZ_LIST \
  X(0,0) X(1,1) X(2,8) X(3,16) X(4,9) X(5,2) X(6,3) X(7,10) X(8,17) X(9,24) X(10,32) X(11,25) X(12,18) X(13,11) X(14,4) X(15,5) \
  X(16,12) X(17,19) X(18,26) X(19,33) X(20,40) X(21,48) X(22,41) X(23,34) X(24,27) X(25,20) X(26,13) X(27,6) X(28,7) X(29,14) X(30,21) X(31,28) \
  X(32,35) X(33,42) X(34,49) X(35,56) X(36,57) X(37,50) X(38,43) X(39,36) X(40,29) X(41,22) X(42,15) X(43,23) X(44,30) X(45,37) X(46,44) X(47,51) \
  X(48,58) X(49,59) X(50,52) X(51,45) X(52,38) X(53,31) X(54,39) X(55,46) X(56,53) X(57,60) X(58,61) X(59,54) X(60,47) X(61,55) X(62,62) X(63,63)

// natural index n (1..63) -> zigzag position, in natural order
#define NAT_LIST Y(1,1) Y(2,5) Y(3,6) Y(4,14) Y(5,15) Y(6,27) Y(7,28) Y(8,2) Y(9,4) Y(10,7) Y(11,13) Y(12,16) Y(13,26) Y(14,29) Y(15,42) Y(16,3) Y(17,8) Y(18,12) Y(19,17) Y(20,25) Y(21,30) Y(22,41) Y(23,43) Y(24,9) Y(25,11) Y(26,18) Y(27,24) Y(28,31) Y(29,40) Y(30,44) Y(31,53) Y(32,10) Y(33,19) Y(34,23) Y(35,32) Y(36,39) Y(37,45) Y(38,52) Y(39,54) Y(40,20) Y(41,22) Y(42,33) Y(43,38) Y(44,46) Y(45,51) Y(46,55) Y(47,60) Y(48,21) Y(49,34) Y(50,37) Y(51,47) Y(52,50) Y(53,56) Y(54,59) Y(55,61) Y(56,35) Y(57,36) Y(58,48) Y(59,49) Y(60,57) Y(61,58) Y(62,62) Y(63,63)

__device__ __forceinline__ int nbits_of(int v) { return 32 - __clz(v); }   // v >= 0 ; JPEG_NBITS (jpeg_nbits.h)

// =====================================================================
// K1: colour conversion + downsampling + deringing + FDCT + quantization
//     one thread per 8x8 block of one component.
//     reference: jccolor.c:213-246 / jccolext.c:30-75, jcsample.c,
//     jcprepct.c:135-192 (edge rules), jcdctmgr.c:416-498,576-604,611-682,
//     693-772, jfdctint.c:142-286.
// =====================================================================
// Component `comp` (in the JPEG colour space) of the pixel at `px`; SB = bytes per sample (1: 8-bit, 2: 12-bit uint16).
//   cs_mode 0: rgb_ycc_convert (jccolext.c:30-75)   1: rgb_gray_convert (Y only)
//           2: null_convert / grayscale_convert (sample `comp`)   3: cmyk_ycck_convert (jccolor.c:395-441)
// first / swap: where the three colour samples sit inside an RGB-family pixel (jccolor.c:253-291, the JCS_EXT_* orders):
// they start at sample `first` and are stored blue-first when `swap` is set; other inputs have first = swap = 0.
// 12-bit samples are masked like the reference's RANGE_LIMIT (jccolext.c:52-54), except YCCK's K, which passes through
// as is (jccolor.c:420).  The fixed-point sums equal the reference's rgb_ycc_tab lookups.
template <int SB>
__device__ __forceinline__ int convert_sample(const uint8_t *__restrict__ px, int cs_mode, int comp, int first, int swap)
{
  constexpr int MAXJ = SB == 1 ? 255 : 4095, CENTRE = (MAXJ + 1) / 2;
  auto smp = [&](int k) -> int { return SB == 1 ? (int)px[k] : (int)(reinterpret_cast<const uint16_t *>(px)[k] & 0xFFF); };
  if (cs_mode == 2 || comp == 3) {                 // component 3 exists in modes 2 and 3 only
    const int k = first + (swap ? 2 - comp : comp);
    return SB == 1 || cs_mode == 2 ? smp(k) : (int)reinterpret_cast<const uint16_t *>(px)[k];
  }
  // cmyk_ycck_convert: R, G, B = MAXJSAMPLE - C, M, Y, which is an XOR for samples in 0..MAXJSAMPLE
  const int inv = cs_mode == 3 ? MAXJ : 0;
  const int r = smp(first + (swap ? 2 : 0)) ^ inv, g = smp(first + 1) ^ inv, b = smp(first + (swap ? 0 : 2)) ^ inv;
  if (comp == 0) return (19595 * r + 38470 * g + 7471 * b + 32768) >> 16;
  if (comp == 1) return (-11059 * r - 21709 * g + 32768 * b + (CENTRE << 16) + 32767) >> 16;
  return (32768 * r - 27439 * g - 5329 * b + (CENTRE << 16) + 32767) >> 16;
}

#define DESCALE(x, n) (((x) + (1 << ((n) - 1))) >> (n))
// P1 = PASS1_BITS: 2 for 8-bit samples, 1 for 12-bit (jfdctint.c:80-86)
template <int PASS, int P1 = 2>
__device__ __forceinline__ void fdct_1d(int &d0, int &d1, int &d2, int &d3, int &d4, int &d5, int &d6, int &d7)
{
  int t0 = d0 + d7, t7 = d0 - d7, t1 = d1 + d6, t6 = d1 - d6;
  int t2 = d2 + d5, t5 = d2 - d5, t3 = d3 + d4, t4 = d3 - d4;
  int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  constexpr int SH = PASS == 0 ? 13 - P1 : 13 + P1;
  if (PASS == 0) { d0 = (t10 + t11) << P1; d4 = (t10 - t11) << P1; }
  else { d0 = DESCALE(t10 + t11, P1); d4 = DESCALE(t10 - t11, P1); }
  int z1 = (t12 + t13) * 4433;
  d2 = DESCALE(z1 + t13 * 6270, SH);
  d6 = DESCALE(z1 + t12 * (-15137), SH);
  z1 = t4 + t7; int z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7;
  int z5 = (z3 + z4) * 9633;
  t4 *= 2446; t5 *= 16819; t6 *= 25172; t7 *= 12299;
  z1 *= -7373; z2 *= -20995; z3 *= -16069; z4 *= -3196;
  z3 += z5; z4 += z5;
  d7 = DESCALE(t4 + z1 + z3, SH);
  d5 = DESCALE(t5 + z2 + z4, SH);
  d3 = DESCALE(t6 + z2 + z3, SH);
  d1 = DESCALE(t7 + z1 + z4, SH);
}

// jcdctmgr.c:387-403 (fp32, no contraction: this TU is built with -fmad=false)
__device__ __forceinline__ float catmull_rom(int v1, int v2, int v3, int v4, float t, int size)
{
  const int tan1 = (v3 - v1) * size, tan2 = (v4 - v2) * size;
  const float t2 = t * t, t3 = t2 * t;
  const float f1 = 2.f * t3 - 3.f * t2 + 1.f;
  const float f2 = -2.f * t3 + 3.f * t2;
  const float f3 = t3 - 2.f * t2 + t;
  const float f4 = t3 - t2;
  return (float)v2 * f1 + (float)tan1 * f3 + (float)v3 * f2 + (float)tan2 * f4;
}
// jcdctmgr.c:416-498 preprocess_deringing on one block; A(n) reads/writes the
// centred sample at NATURAL index n.  Rare path (blocks touching max white).
template <class Acc>
__device__ __forceinline__ void deringing_block(Acc A, int q0, int sum, int cnt)
{
  const int maxsample = 127, size = 64;
  int m = min(min(31, 2 * q0), (maxsample * size - sum) / cnt);
  int maxover = maxsample + m;
  int n = 0;
  do {
    if (A.get(c_zz[n]) < maxsample) { n++; continue; }
    int start = n;
    while (++n < size && A.get(c_zz[n]) >= maxsample) {}
    int end = n;
    int f1 = A.get(c_zz[start >= 1 ? start - 1 : 0]);
    int f2 = A.get(c_zz[start >= 2 ? start - 2 : 0]);
    int l1 = A.get(c_zz[end < size - 1 ? end : size - 1]);
    int l2 = A.get(c_zz[end < size - 2 ? end + 1 : size - 1]);
    int fslope = max(f1 - f2, maxsample - f1);
    int lslope = max(l1 - l2, maxsample - l1);
    if (start == 0) fslope = lslope;
    if (end == size) lslope = fslope;
    int length = end - start;
    float step = 1.f / (float)(length + 1);
    float position = step;
    for (int i = start; i < end; i++, position += step) {
      int tmp = (int)ceilf(catmull_rom(maxsample - fslope, maxsample, maxsample, maxsample - lslope, position, length));
      A.set(c_zz[i], min(tmp, maxover));
    }
    n++;
  } while (n < size);
}
struct LocalAcc { int *d; __device__ int get(int n) const { return d[n]; } __device__ void set(int n, int v) const { d[n] = v; } };
struct PlaneAcc {      // 8x8 block inside an int16 sample plane in shared memory
  int16_t *p; int pitch;
  __device__ int get(int n) const { return p[(n >> 3) * pitch + (n & 7)]; }
  __device__ void set(int n, int v) const { p[(n >> 3) * pitch + (n & 7)] = (int16_t)v; }
};

__device__ __forceinline__ unsigned quant_one(int x, QuantConst k, int dering)
{
  unsigned a = (unsigned)abs(x) + k.bias;
  int q = (int)(((unsigned long long)a * k.mul) >> k.shift);
  if (dering) q = min(q, 1023);            // (1 << (8 + 2)) - 1
  return (unsigned)(x < 0 ? -q : q);
}

// ---- JDCT_IFAST (jfdctfst.c:113-224): MULTIPLY = (v * c) >> 8, no rounding ----
__device__ __forceinline__ void fdct_ifast_1d(int &d0, int &d1, int &d2, int &d3, int &d4, int &d5, int &d6, int &d7)
{
  int tmp0 = d0 + d7, tmp7 = d0 - d7, tmp1 = d1 + d6, tmp6 = d1 - d6;
  int tmp2 = d2 + d5, tmp5 = d2 - d5, tmp3 = d3 + d4, tmp4 = d3 - d4;
  int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  d0 = tmp10 + tmp11; d4 = tmp10 - tmp11;
  int z1 = ((tmp12 + tmp13) * 181) >> 8;
  d2 = tmp13 + z1; d6 = tmp13 - z1;
  tmp10 = tmp4 + tmp5; tmp11 = tmp5 + tmp6; tmp12 = tmp6 + tmp7;
  int z5 = ((tmp10 - tmp12) * 98) >> 8;
  int z2 = ((tmp10 * 139) >> 8) + z5;
  int z4 = ((tmp12 * 334) >> 8) + z5;
  int z3 = (tmp11 * 181) >> 8;
  int z11 = tmp7 + z3, z13 = tmp7 - z3;
  d5 = z13 + z2; d3 = z13 - z2; d1 = z11 + z4; d7 = z11 - z4;
}
__constant__ short c_aanscales[64] = {
  16384, 22725, 21407, 19266, 16384, 12873,  8867,  4520,
  22725, 31521, 29692, 26722, 22725, 17855, 12299,  6270,
  21407, 29692, 27969, 25172, 21407, 16819, 11585,  5906,
  19266, 26722, 25172, 22654, 19266, 15137, 10426,  5315,
  16384, 22725, 21407, 19266, 16384, 12873,  8867,  4520,
  12873, 17855, 16819, 15137, 12873, 10114,  6967,  3552,
   8867, 12299, 11585, 10426,  8867,  6967,  4799,  2446,
   4520,  6270,  5906,  5315,  4520,  3552,  2446,  1247};

// ---- JDCT_FLOAT (jfdctflt.c:59-167, AA&N): one 1-D pass, fp32, no contraction ----
__device__ __forceinline__ void fdct_float_1d(float &d0, float &d1, float &d2, float &d3, float &d4, float &d5, float &d6, float &d7)
{
  float tmp0 = d0 + d7, tmp7 = d0 - d7, tmp1 = d1 + d6, tmp6 = d1 - d6;
  float tmp2 = d2 + d5, tmp5 = d2 - d5, tmp3 = d3 + d4, tmp4 = d3 - d4;
  float tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  d0 = tmp10 + tmp11; d4 = tmp10 - tmp11;
  float z1 = (tmp12 + tmp13) * 0.707106781f;
  d2 = tmp13 + z1; d6 = tmp13 - z1;
  tmp10 = tmp4 + tmp5; tmp11 = tmp5 + tmp6; tmp12 = tmp6 + tmp7;
  float z5 = (tmp10 - tmp12) * 0.382683433f;
  float z2 = 0.541196100f * tmp10 + z5;
  float z4 = 1.306562965f * tmp12 + z5;
  float z3 = tmp11 * 0.707106781f;
  float z11 = tmp7 + z3, z13 = tmp7 - z3;
  d5 = z13 + z2; d3 = z13 - z2; d1 = z11 + z4; d7 = z11 - z4;
}
// float_preprocess_deringing (jcdctmgr.c:503-575) on 64 floats in natural order; catmull_rom takes DCTELEM (int)
// values, so the float slopes are truncated on the way in
__device__ __forceinline__ void deringing_block_float(float *data, int q0, float sum, int cnt)
{
  const float maxsample = 127.0f; const int size = 64;
  const int a = min(31, 2 * q0); const float bq = (maxsample * size - sum) / (float)cnt;
  const float maxovershoot = maxsample + ((float)a < bq ? (float)a : bq);
  int n = 0;
  do {
    if (data[c_zz[n]] < maxsample) { n++; continue; }
    int start = n;
    while (++n < size && data[c_zz[n]] >= maxsample) {}
    int end = n;
    float f1 = data[c_zz[start >= 1 ? start - 1 : 0]], f2 = data[c_zz[start >= 2 ? start - 2 : 0]];
    float l1 = data[c_zz[end < size - 1 ? end : size - 1]], l2 = data[c_zz[end < size - 2 ? end + 1 : size - 1]];
    float fslope = fmaxf(f1 - f2, maxsample - f1), lslope = fmaxf(l1 - l2, maxsample - l1);
    if (start == 0) fslope = lslope;
    if (end == size) lslope = fslope;
    int length = end - start;
    float step = 1.f / (float)(length + 1), position = step;
    for (int i = start; i < end; i++, position += step) {
      float tmp = catmull_rom((int)(maxsample - fslope), 127, 127, (int)(maxsample - lslope), position, length);
      data[c_zz[i]] = tmp < maxovershoot ? tmp : maxovershoot;
    }
    n++;
  } while (n < size);
}
__constant__ double c_aan[8] = {1.0, 1.387039845, 1.306562965, 1.175875602, 1.0, 0.785694958, 0.541196100, 0.275899379};

// PREC: 8 or 12 (uint16 samples); DCTM: 0 = JDCT_ISLOW, 1 = JDCT_IFAST, 2 = JDCT_FLOAT; same arithmetic as the tiled
// kernel's paths, plus the 12-bit forms of the fast and the float DCT.
__device__ __forceinline__ unsigned qc_d(const QuantTables *__restrict__ qt, int t, int i) { return qt->q[t][i].d; }   // 8 * quantval
template <int PREC, int DCTM>
__global__ void __launch_bounds__(128) k_forward(Geom g, const uint8_t *__restrict__ src,
                                                 const QuantTables *__restrict__ qt, int dering,
                                                 DcRec *__restrict__ rec, RecLayout rl)
{
  constexpr int CENTRE = 1 << (PREC - 1);
  constexpr int SB = PREC == 8 ? 1 : 2;
  constexpr int P1 = PREC == 8 ? 2 : 1;                  // PASS1_BITS (jfdctint.c:80-86)
  const int ci = blockIdx.z % g.nc, img = blockIdx.z / g.nc;
  const CompGeom &c = g.c[ci];
  int bx = blockIdx.x * blockDim.x + threadIdx.x;
  int by = blockIdx.y;
  if (bx >= c.wib || by >= c.hib) return;
  // the image's table set, re-derived at each use (a pointer held across the kernel costs spills)
  auto set = [&] { return qset_of(qt, g, img); };
  const uint8_t *base = src + (size_t)img * g.image_stride;
  int ws[64];
  const int comp = g.cs_mode == 1 ? 0 : ci;
  auto component = [&](const uint8_t *px) -> int { return convert_sample<SB>(px, g.cs_mode, comp, g.px_first, g.px_swap); };
#pragma unroll
  for (int y = 0; y < 8; y++) {
    int yo = by * 8 + y;
    int yy = min(yo, c.rows_avail - 1);                   // expand_bottom_edge on downsampled rows
    int grp = yy / c.v, sub = yy - grp * c.v;
    int iy0 = grp * g.vmax + sub * c.vx;
#pragma unroll
    for (int x = 0; x < 8; x++) {
      int xo = bx * 8 + x;
      if (g.raw_in) {                                     // component planes (raw-data input / the smoothing pre-pass): only centre them
        const uint8_t *q = g.plane[ci] + (size_t)img * g.plane_stride[ci] + (size_t)yo * g.plane_pitch[ci] + (size_t)xo * SB;
        ws[8 * y + x] = (SB == 1 ? (int)*q : (int)*reinterpret_cast<const uint16_t *>(q)) - CENTRE;
        continue;
      }
      int sum = 0;
      for (int dv = 0; dv < c.vx; dv++) {
        int iy = min(iy0 + dv, g.H - 1);                  // bottom row replication inside the row group
        const uint8_t *row = base + (size_t)iy * g.row_pitch;
        for (int du = 0; du < c.hx; du++) {
          int ix = min(xo * c.hx + du, g.W - 1);          // expand_right_edge (jcsample.c:98-116)
          sum += component(row + (size_t)ix * g.in_comps * SB);
        }
      }
      int val;
      if (c.hx == 1 && c.vx == 1) val = sum;
      else if (c.hx == 2 && c.vx == 1) val = (sum + (xo & 1)) >> 1;          // jcsample.c:226-254
      else if (c.hx == 2 && c.vx == 2) val = (sum + 1 + (xo & 1)) >> 2;      // jcsample.c:263-295
      else { int np = c.hx * c.vx; val = (sum + np / 2) / np; }              // jcsample.c:151-190
      ws[8 * y + x] = val - CENTRE;                                          // convsamp
    }
  }
  int qv[64];                                              // quantized values, natural order (fast / float DCT)
  if (DCTM == 2) {
    // convsamp_float -> float deringing -> jpeg_fdct_float -> quantize_float + the trellis' integer coefficients
    float wf[64];
    int sum = 0, cnt = 0;
#pragma unroll
    for (int i = 0; i < 64; i++) { wf[i] = (float)ws[i]; sum += ws[i]; cnt += (ws[i] >= 127); }
    if (dering && cnt != 0 && cnt != 64) deringing_block_float(wf, (int)set()->q[c.qt][0].d >> 3, (float)sum, cnt);
#pragma unroll
    for (int r = 0; r < 8; r++) fdct_float_1d(wf[8 * r], wf[8 * r + 1], wf[8 * r + 2], wf[8 * r + 3], wf[8 * r + 4], wf[8 * r + 5], wf[8 * r + 6], wf[8 * r + 7]);
#pragma unroll
    for (int col = 0; col < 8; col++) fdct_float_1d(wf[col], wf[8 + col], wf[16 + col], wf[24 + col], wf[32 + col], wf[40 + col], wf[48 + col], wf[56 + col]);
    const float *fd = set()->fdiv[c.qt];
#pragma unroll
    for (int i = 0; i < 64; i++) {
      float v = wf[i];
      v = (float)((double)v / c_aan[i & 7]);               // forward_DCT_float :860-874
      v = (float)((double)v / c_aan[i >> 3]);
      ws[i] = (v >= 0.0f) ? (int)((double)v + 0.5) : (int)((double)v - 0.5);
      int q = (int)(int16_t)(__float2int_rz(wf[i] * fd[i] + 16384.5f) - 16384);     // quantize_float :808-827
      if (dering) q = max(-1023, min(1023, q));
      qv[i] = q;
    }
  } else {
    if (dering) {
      int sum = 0, cnt = 0;
#pragma unroll
      for (int i = 0; i < 64; i++) { sum += ws[i]; cnt += (ws[i] >= 127); }
      if (cnt != 0 && cnt != 64) {
        int tmp[64];
#pragma unroll
        for (int i = 0; i < 64; i++) tmp[i] = ws[i];
        deringing_block(LocalAcc{tmp}, (int)set()->q[c.qt][0].d >> 3, sum, cnt);
#pragma unroll
        for (int i = 0; i < 64; i++) ws[i] = tmp[i];
      }
    }
    if (DCTM == 1) {
#pragma unroll
      for (int r = 0; r < 8; r++) fdct_ifast_1d(ws[8 * r], ws[8 * r + 1], ws[8 * r + 2], ws[8 * r + 3], ws[8 * r + 4], ws[8 * r + 5], ws[8 * r + 6], ws[8 * r + 7]);
#pragma unroll
      for (int col = 0; col < 8; col++) fdct_ifast_1d(ws[col], ws[8 + col], ws[16 + col], ws[24 + col], ws[32 + col], ws[40 + col], ws[48 + col], ws[56 + col]);
      const IfastConst *ic = set()->ifast[c.qt];
#pragma unroll
      for (int i = 0; i < 64; i++) {
        const int x = ws[i], sc = c_aanscales[i];
        const int a = abs(x);
        int q;
        if (PREC == 8) {
          const IfastConst k = ic[i];                       // reciprocal quantizer of jcdctmgr.c:611-645 on the scaled divisor
          q = (int)(int16_t)(int)(((unsigned long long)(unsigned)(a + (int)k.corr) * k.recip) >> (k.shift + 32));
        } else {
          // 12-bit build: the scaled divisor stays a JLONG (jcdctmgr.c:332-336) and quantize() divides literally (:646-678)
          const int d = (int)(((long long)((int)qc_d(set(), c.qt, i) >> 3) * sc + (1 << 10)) >> 11);
          q = (int)(int16_t)((a + (d >> 1)) / d);
        }
        if (x < 0) q = (int)(int16_t)(-q);
        if (dering) q = max(-1023, min(1023, q));
        qv[i] = q;
        ws[i] = (int)((x >= 0) ? ((long long)x * 32768 + sc) / (2 * sc) : ((long long)x * 32768 - sc) / (2 * sc));     // the trellis' coefficient (jcdctmgr.c:729-746)
      }
    } else {
#pragma unroll
      for (int r = 0; r < 8; r++)
        fdct_1d<0, P1>(ws[8 * r], ws[8 * r + 1], ws[8 * r + 2], ws[8 * r + 3], ws[8 * r + 4], ws[8 * r + 5], ws[8 * r + 6], ws[8 * r + 7]);
#pragma unroll
      for (int col = 0; col < 8; col++)
        fdct_1d<1, P1>(ws[col], ws[8 + col], ws[16 + col], ws[24 + col], ws[32 + col], ws[40 + col], ws[48 + col], ws[56 + col]);
    }
  }
  const QuantConst *qc = set()->q[c.qt];
  if (rec) {       // side record for the trellis: norm numerator in natural order (jcdctmgr.c:1026-1029), raw DC, #non-zero ACs
    float norm = 0.0f; unsigned long long mask = 0;
#pragma unroll
    for (int i = 1; i < 64; i++) {
      norm += (float)(ws[i] * ws[i]);
      // the trellis derives its entries from the RAW coefficient (qval = (|x| + q/2) / q, jcdctmgr.c:1136)
      bool nz;
      if (DCTM == 0) nz = quant_one(ws[i], qc[i], dering) != 0u;
      else { const int dq = (int)qc[i].d; nz = abs(ws[i]) >= dq - dq / 2; }
      if (nz) mask |= 1ull << c_izz[i];
    }
    DcRec rr; rr.lambda_dc = norm; rr.raw_dc = (int16_t)ws[0]; rr.nz = (uint8_t)__popcll(mask); rr.pad = 0; rr.nzmask = mask;
    rec[(size_t)img * rl.per_image + rl.comp_off[ci] + (size_t)by * c.wib + bx] = rr;
  }
  // quantize (jcdctmgr.c:611-682 == sign(x)*floor((|x| + d/2)/d), d = 8Q) + deringing clamp (:761-770),
  // packed two int16 per 32-bit word in ZIGZAG order
  size_t blk = ((size_t)img * c.hpad + by) * c.wpad + bx;
  uint4 *dq = reinterpret_cast<uint4 *>(c.coef + blk * 64);
  uint4 *dr = reinterpret_cast<uint4 *>(c.raw + blk * 64);
  unsigned pq[32], pr[32];
#define X(k, n) { unsigned qq = (DCTM == 0 ? quant_one(ws[n], qc[n], dering) : (unsigned)qv[n]) & 0xFFFFu, rr = (unsigned)ws[n] & 0xFFFFu; \
                  if ((k) & 1) { pq[(k) >> 1] |= qq << 16; pr[(k) >> 1] |= rr << 16; } else { pq[(k) >> 1] = qq; pr[(k) >> 1] = rr; } }
  ZZ_LIST
#undef X
#pragma unroll
  for (int v = 0; v < 8; v++) {
    dq[v] = make_uint4(pq[4 * v], pq[4 * v + 1], pq[4 * v + 2], pq[4 * v + 3]);
    dr[v] = make_uint4(pr[4 * v], pr[4 * v + 1], pr[4 * v + 2], pr[4 * v + 3]);
  }
}

// =====================================================================
// K1, tiled fast path (the common layouts: RGB->YCbCr with full-size luma
// and 1x1-sampled chroma, i.e. 4:4:4 / 4:2:2 / 4:4:0 / 4:2:0, and grayscale).
// One CTA = one strip of an iMCU row, 128 pixels wide:
//   A. coalesced 16-byte loads of the RGB strip into shared memory;
//   B. colour conversion + box downsampling into int16 sample planes (smem);
//   C. 8 threads per 8x8 block: row pass of the FDCT (after the deringing
//      pre-filter), transposed through shared memory;
//   D. column pass, quantization, zigzag placement into a staging buffer;
//   E. coalesced 16-byte stores of whole 128-byte blocks.
// Same arithmetic as k_forward (the generic one-thread-per-block kernel).
// =====================================================================
template <int PREC> struct WorkT { typedef int16_t type; };
template <> struct WorkT<12> { typedef int type; };
template <> struct WorkT<32> { typedef float type; };
// One row of 8 pixels of the strip in registers: IC samples per pixel, SB bytes per sample
// (8-bit: 24 bytes RGB / 8 grey; 12-bit in uint16: 48 / 16).
struct Px8 { unsigned w[12]; };
// px4: the pixels in memory have 4 samples (JCS_EXT_RGBX/BGRX/XBGR/XRGB and the alpha orders); the three colour samples
// start at sample `first` (0 or 1) and are packed to the 3-sample register layout on the way in
template <int IC, int SB>
__device__ __forceinline__ Px8 load_px8(const uint8_t *__restrict__ base, size_t row_pitch, int iy, int x, int W, bool fast, bool px4 = false, int first = 0)
{
  Px8 r;
  const uint8_t *row = base + (size_t)iy * row_pitch;
  constexpr int NBYTES = 8 * IC * SB;
#pragma unroll
  for (int i = 0; i < 12; i++) r.w[i] = 0;
  if (fast && IC == 3 && px4) {
    // 8 pixels x 4 samples, aligned: drop the filler sample (byte permutes; a 16-bit sample is two bytes)
    unsigned q[16];
    if (SB == 1) {
      const uint4 *p = reinterpret_cast<const uint4 *>(row + (size_t)x * 4);
      const uint4 a = __ldg(p), b = __ldg(p + 1);
      q[0] = a.x; q[1] = a.y; q[2] = a.z; q[3] = a.w; q[4] = b.x; q[5] = b.y; q[6] = b.z; q[7] = b.w;
      if (first) {
#pragma unroll
        for (int i = 0; i < 8; i++) q[i] >>= 8;                    // colour samples into bytes 0..2
      }
#pragma unroll
      for (int g4 = 0; g4 < 2; g4++) {                             // 4 pixels (12 bytes) per group
        const unsigned p0 = q[4 * g4], p1 = q[4 * g4 + 1], p2 = q[4 * g4 + 2], p3 = q[4 * g4 + 3];
        r.w[3 * g4] = __byte_perm(p0, p1, 0x4210);
        r.w[3 * g4 + 1] = __byte_perm(p1, p2, 0x5421);
        r.w[3 * g4 + 2] = __byte_perm(p2, p3, 0x6542);
      }
    } else {
      const uint4 *p = reinterpret_cast<const uint4 *>(row + (size_t)x * 8);
#pragma unroll
      for (int i = 0; i < 4; i++) { const uint4 a = __ldg(p + i); q[4 * i] = a.x; q[4 * i + 1] = a.y; q[4 * i + 2] = a.z; q[4 * i + 3] = a.w; }
      // pixel k = words 2k, 2k+1 (4 halfwords); output halfword h = 3k + c <- pixel k, halfword first + c
#pragma unroll
      for (int k = 0; k < 8; k++) {
        const unsigned lo = q[2 * k], hi = q[2 * k + 1];
        const unsigned c0 = first ? (lo >> 16) : (lo & 0xFFFFu), c1 = first ? (hi & 0xFFFFu) : (lo >> 16), c2 = first ? (hi >> 16) : (hi & 0xFFFFu);
        const unsigned cc[3] = {c0, c1, c2};
#pragma unroll
        for (int c = 0; c < 3; c++) { const int h = 3 * k + c; r.w[h >> 1] |= cc[c] << (16 * (h & 1)); }
      }
    }
    return r;
  }
  if (fast) {                                     // aligned (8 bytes for 8-bit, 16 for 16-bit samples), fully inside the image
    if (SB == 1) {
      const uint2 *p = reinterpret_cast<const uint2 *>(row + (size_t)x * IC);
#pragma unroll
      for (int i = 0; i < NBYTES / 8; i++) { uint2 a = __ldg(p + i); r.w[2 * i] = a.x; r.w[2 * i + 1] = a.y; }
    } else {
      const uint4 *p = reinterpret_cast<const uint4 *>(row + (size_t)x * IC * 2);
#pragma unroll
      for (int i = 0; i < NBYTES / 16; i++) { uint4 a = __ldg(p + i); r.w[4 * i] = a.x; r.w[4 * i + 1] = a.y; r.w[4 * i + 2] = a.z; r.w[4 * i + 3] = a.w; }
    }
  } else {                                        // right edge / unaligned: bytes, columns clamped to W-1 (expand_right_edge)
    const int pxb = (IC == 3 && px4 ? 4 : IC) * SB, off = (IC == 3 && px4 ? first : 0) * SB;
#pragma unroll
    for (int b = 0; b < NBYTES; b++) {
      int px = b / (IC * SB), rem = b - px * (IC * SB);
      int ix = min(x + px, W - 1);
      r.w[b >> 2] |= (unsigned)row[(size_t)ix * pxb + off + rem] << (8 * (b & 3));
    }
  }
  return r;
}
// sample `ch` of pixel `px`; 12-bit samples are masked like the reference's RANGE_LIMIT (jccolext.c:52-54)
template <int IC, int SB>
__device__ __forceinline__ int px_sample(const Px8 &r, int px, int ch)
{
  if (SB == 1) { int b = px * IC + ch; return (int)__byte_perm(r.w[b >> 2], 0u, 0x4440 | (b & 3)); }   // byte b of the packed row (one PRMT)
  int h = px * IC + ch; return (int)((r.w[h >> 1] >> (16 * (h & 1))) & 0xFFFu);
}

// exact floor((|x| + d/2) / d) * sign(x) with the per-table uniform shift (QuantTables.fast) or the general 64-bit form
__device__ __forceinline__ int quant_fast(int x, uint2 k, int L, int dering)
{
  unsigned a14 = (unsigned)abs(x) * 16384u + k.y;            // (|x| + d/2) << 14   (< 2^32)
  int q = (int)(__umulhi(a14, k.x) >> L);
  if (dering) q = min(q, 1023);                              // (1 << (8 + 2)) - 1
  return x < 0 ? -q : q;
}


// DCTM: 0 = JDCT_ISLOW, 1 = JDCT_IFAST, 2 = JDCT_FLOAT (1 and 2: 8-bit only in this kernel; 12-bit: k_forward)
#ifndef FWD_MASK_SQ
#define FWD_MASK_SQ 1
#endif
#ifndef FWD_MIN_CTAS
#define FWD_MIN_CTAS 6
#endif
template <int HMAX, int VMAX, int NC, bool QFAST, int PREC, int DCTM>
__global__ void __launch_bounds__(128, FWD_MIN_CTAS) k_forward_tile(Geom g, const uint8_t *__restrict__ src,
                                                      const QuantTables *__restrict__ qt, int dering,
                                                      DcRec *__restrict__ rec, RecLayout rl, int write_raw, FwdStats fs,
                                                      const __grid_constant__ CUtensorMap tmap, const int use_tma)
{
  constexpr int TW = 128, TR = 8 * VMAX;
  constexpr int YBW = TW / 8, YB = YBW * VMAX;           // luma blocks in the tile
  constexpr int CW = TW / HMAX, CBW = CW / 8;            // chroma samples / blocks per tile row
  constexpr int NB = YB + (NC == 3 ? 2 * CBW : 0);
  constexpr int YP = TW + 8, CP = CW + 8;                // padded plane pitches (int16 elements)
  constexpr int IC = NC == 3 ? 3 : 1;                    // samples per input pixel on the fast path (grey from RGB: see below)
  constexpr int SB = PREC == 8 ? 1 : 2;                  // bytes per sample (12-bit samples come as uint16)
  constexpr int P1 = PREC == 8 ? 2 : 1;                  // PASS1_BITS
  constexpr int CENTRE = 1 << (PREC - 1);
  typedef typename WorkT<DCTM == 2 ? 32 : PREC>::type wtype;   // row-pass results: int16 holds them at 8 bits, int32 at 12, float for JDCT_FLOAT
  __shared__ __align__(16) int16_t sY[TR * YP];
  __shared__ __align__(16) int16_t sC[NC == 3 ? 2 * 8 * CP : 8];
  __shared__ __align__(16) wtype sW[NB * 72];
  __shared__ __align__(128) unsigned char sIO[NB * 256];  // phase A: the tile's pixels as the TMA delivers them; phases D/E: output staging
  __shared__ __align__(8) unsigned long long tma_bar;
  __shared__ __align__(16) uint2 sQC[NC][64];            // quantizer constants per component, natural order
  __shared__ uint2 sMask[NB];                             // per block: zigzag positions of its non-zero AC values
  __shared__ int sQL[NC];
  constexpr int HW4 = (HIST_BINS + 3) / 4;                 // 16-byte words per histogram (the padding bins stay 0)
  __shared__ __align__(16) unsigned sHist[NC][4 * HW4];    // fs.hist: the tile's AC symbol counts per component

  const int tid = threadIdx.x;
  const int tx = blockIdx.x, ty = blockIdx.y, img = blockIdx.z;
  const int x0 = tx * TW, y0 = ty * TR;
  const uint8_t *base = src + (size_t)img * g.image_stride;
  qt = qset_of(qt, g, img);

  // ---- A0: interior tiles of 8-bit RGB / gray input arrive by TMA: one thread posts the tile's box(es) of the
  //      (bytes per row, rows, images) tensor map -- 128 pixels x TR rows, 192-byte boxes because a box dimension is
  //      capped at 256 elements -- and everybody waits on the mbarrier the copies complete on.  Edge tiles (pixel
  //      replication) and unaligned inputs keep the per-thread global loads.  The copy is posted first, so that the
  //      quantizer constants and the histogram clear below run while it is in flight. ----
  constexpr int TMA_BOXW = IC == 3 ? 192 : 128, TMA_NBOX = IC == 3 ? 2 : 1;
  static_assert(TMA_NBOX * TMA_BOXW * TR <= NB * 256, "the pixel tile fits the staging buffer it borrows");
  const bool tma_tile = PREC == 8 && use_tma && x0 + TW <= g.W && y0 + TR <= g.H;
  const unsigned bar = (unsigned)__cvta_generic_to_shared(&tma_bar);
  if (tma_tile && tid == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(bar) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"((unsigned)(TMA_NBOX * TMA_BOXW * TR)) : "memory");
#pragma unroll
    for (int bx = 0; bx < TMA_NBOX; bx++)
      asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                   :: "r"((unsigned)__cvta_generic_to_shared(sIO + bx * TMA_BOXW * TR)), "l"(reinterpret_cast<unsigned long long>(&tmap)),
                      "r"(x0 * IC + bx * TMA_BOXW), "r"(y0), "r"(g.image_stride ? img : 0), "r"(bar) : "memory");   // stride 0: one image for all
  }

  if (fs.hist) for (int i = tid; i < NC * HW4; i += 128) reinterpret_cast<uint4 *>(&sHist[0][0])[i] = make_uint4(0, 0, 0, 0);
  // the packed {mul2, bias << 14} pairs, built once per table set on the host (QuantTables.qpack): 16-byte copies
  if (QFAST && DCTM == 0)                                    // the only quantizer that reads them
    for (int i = tid; i < NC * 32; i += 128)
      reinterpret_cast<uint4 *>(sQC[i >> 5])[i & 31] = reinterpret_cast<const uint4 *>(qt->qpack[g.c[i >> 5].qt])[i & 31];
  if (tid < NC) sQL[tid] = qt->L[g.c[tid].qt];

  if (tma_tile) {
    __syncthreads();                                             // the barrier word is initialised before anyone polls it
    {
      unsigned done = 0;
      while (!done)
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0; selp.u32 %0, 1, 0, p; }" : "=r"(done) : "r"(bar) : "memory");
    }
  }

  // ---- A+B: thread (row group rg, segment seg) converts VMAX rows x 8 pixels (from the TMA tile or straight from
  //      global memory): colour conversion (jccolext.c:30-75) + box downsampling (jcsample.c) into centred int16 planes ----
  {
    const int rg = tid >> 4, seg = tid & 15;
    const int xs = x0 + seg * 8;
    // this thread's 8 pixels of tile row `trow` out of the TMA tile
    auto tma_px8 = [&](int trow) {
      Px8 r;
#pragma unroll
      for (int i = 0; i < 12; i++) r.w[i] = 0;
      if (IC == 3) {
        const uint2 *q = reinterpret_cast<const uint2 *>(sIO + (seg >> 3) * (TMA_BOXW * TR) + trow * TMA_BOXW + (seg & 7) * 24);
#pragma unroll
        for (int i = 0; i < 3; i++) { const uint2 a = q[i]; r.w[2 * i] = a.x; r.w[2 * i + 1] = a.y; }
      } else {
        const uint2 a = *reinterpret_cast<const uint2 *>(sIO + trow * TMA_BOXW + seg * 8);
        r.w[0] = a.x; r.w[1] = a.y;
      }
      return r;
    };
    if (g.raw_in) {
      // raw-data input: the planes are already converted and downsampled; only centre them (convsamp).  Samples past
      // the component's last real block are never used (those blocks are skipped on output), so they read as 0.
      // Plane pitches and strides are in bytes; 12-bit planes (the smoothing pre-pass makes them) hold uint16 samples.
      auto sample = [&](int cc, int row, int x) -> int {
        const uint8_t *q = g.plane[cc] + (size_t)img * g.plane_stride[cc] + (size_t)row * g.plane_pitch[cc] + (size_t)x * SB;
        return SB == 1 ? (int)*q : (int)*reinterpret_cast<const uint16_t *>(q);
      };
#pragma unroll
      for (int rr = 0; rr < VMAX; rr++) {
        const int row = y0 + rg * VMAX + rr;
        const CompGeom &c0 = g.c[0];
        int16_t yv[8];
#pragma unroll
        for (int px = 0; px < 8; px++) {
          const int x = xs + px;
          yv[px] = (row < c0.hib * 8 && x < c0.wib * 8) ? (int16_t)(sample(0, row, x) - CENTRE) : (int16_t)0;
        }
        *reinterpret_cast<uint4 *>(&sY[(rg * VMAX + rr) * YP + seg * 8]) = *reinterpret_cast<const uint4 *>(yv);
      }
      if (NC == 3) {
        const int row = ty * 8 + rg;
#pragma unroll
        for (int cc = 1; cc <= 2; cc++) {
          const CompGeom &c1 = g.c[cc];
          int16_t cv[8 / HMAX];
#pragma unroll
          for (int i = 0; i < 8 / HMAX; i++) {
            const int x = x0 / HMAX + seg * (8 / HMAX) + i;
            cv[i] = (row < c1.hib * 8 && x < c1.wib * 8) ? (int16_t)(sample(cc, row, x) - CENTRE) : (int16_t)0;
          }
          int16_t *dst = &sC[(cc - 1) * 8 * CP + rg * CP + seg * (8 / HMAX)];
          if (HMAX == 1) *reinterpret_cast<uint4 *>(dst) = *reinterpret_cast<const uint4 *>(cv);
          else *reinterpret_cast<uint2 *>(dst) = *reinterpret_cast<const uint2 *>(cv);
        }
      }
    } else {
    const bool grey_from_rgb = NC == 1 && g.cs_mode == 1;
    const bool px4 = g.in_comps == 4 && (NC == 3 || grey_from_rgb);       // 4-sample RGB-family pixels
    const int pfirst = g.px_first; const bool pswap = g.px_swap != 0;
    const size_t AL = px4 ? 15 : (SB == 1 ? 7 : 15);
    const bool fast = (xs + 8 <= g.W) && ((g.row_pitch & AL) == 0) && ((((size_t)base) & AL) == 0) && !grey_from_rgb;
    if (NC == 1 && grey_from_rgb) {
      // RGB input, grayscale output: 3 bytes per pixel, luma only
#pragma unroll
      for (int rr = 0; rr < VMAX; rr++) {
        const int iy = min(y0 + rg * VMAX + rr, g.H - 1);
        const bool f3 = (xs + 8 <= g.W) && ((g.row_pitch & AL) == 0) && ((((size_t)base) & AL) == 0);
        Px8 p = load_px8<3, SB>(base, g.row_pitch, iy, xs, g.W, f3, px4, pfirst);
        int16_t yv[8];
#pragma unroll
        for (int px = 0; px < 8; px++) {
          const int s0 = px_sample<3, SB>(p, px, 0), s2 = px_sample<3, SB>(p, px, 2);
          yv[px] = (int16_t)(((19595 * (pswap ? s2 : s0) + 38470 * px_sample<3, SB>(p, px, 1) + 7471 * (pswap ? s0 : s2) + 32768) >> 16) - CENTRE);
        }
        *reinterpret_cast<uint4 *>(&sY[(rg * VMAX + rr) * YP + seg * 8]) = *reinterpret_cast<const uint4 *>(yv);
      }
    } else {
      // EXT: the input is one of the other pixel orders (4-sample pixels and / or blue first); the plain RGB / YCbCr /
      // gray instantiation carries none of that logic
      auto convert = [&](auto ext_tag) {
      constexpr bool EXT = decltype(ext_tag)::value;
      int sb[8 / HMAX], sr[8 / HMAX];
#pragma unroll
      for (int i = 0; i < 8 / HMAX; i++) { sb[i] = 0; sr[i] = 0; }
      // chroma rows past the last real row group replicate the last real chroma row (jcprepct.c:167-179)
      const int last_real = NC == 3 ? g.c[1].rows_avail - 1 - ty * 8 : 8;
      const int er = min(rg, last_real);
#pragma unroll
      for (int rr = 0; rr < VMAX; rr++) {
        const int iy = min(y0 + rg * VMAX + rr, g.H - 1);
        Px8 p = (!EXT && tma_tile) ? tma_px8(rg * VMAX + rr) : load_px8<IC, SB>(base, g.row_pitch, iy, xs, g.W, fast, EXT && px4, EXT ? pfirst : 0);
        int16_t yv[8];
#pragma unroll
        for (int px = 0; px < 8; px++) {
          if (NC == 1) yv[px] = (int16_t)(px_sample<1, SB>(p, px, 0) - CENTRE);
          else {
            const int S0 = px_sample<3, SB>(p, px, 0), G = px_sample<3, SB>(p, px, 1), S2 = px_sample<3, SB>(p, px, 2);
            const int R = (EXT && pswap) ? S2 : S0, B = (EXT && pswap) ? S0 : S2;
            yv[px] = (int16_t)(((19595 * R + 38470 * G + 7471 * B + 32768) >> 16) - CENTRE);
          }
        }
        *reinterpret_cast<uint4 *>(&sY[(rg * VMAX + rr) * YP + seg * 8]) = *reinterpret_cast<const uint4 *>(yv);
        if (NC == 3) {
          if (er != rg) p = (!EXT && tma_tile) ? tma_px8(er * VMAX + rr) : load_px8<IC, SB>(base, g.row_pitch, min(y0 + er * VMAX + rr, g.H - 1), xs, g.W, fast, EXT && px4, EXT ? pfirst : 0);
#pragma unroll
          for (int px = 0; px < 8; px++) {
            const int S0 = px_sample<3, SB>(p, px, 0), G = px_sample<3, SB>(p, px, 1), S2 = px_sample<3, SB>(p, px, 2);
            const int R = (EXT && pswap) ? S2 : S0, B = (EXT && pswap) ? S0 : S2;
            sb[px / HMAX] += (-11059 * R - 21709 * G + 32768 * B + (CENTRE << 16) + 32767) >> 16;
            sr[px / HMAX] += (32768 * R - 27439 * G - 5329 * B + (CENTRE << 16) + 32767) >> 16;
          }
        }
      }
      if (NC == 3) {
        int16_t cbv[8 / HMAX], crv[8 / HMAX];
#pragma unroll
        for (int i = 0; i < 8 / HMAX; i++) {
          const int xo = x0 / HMAX + seg * (8 / HMAX) + i;
          int b = sb[i], r = sr[i];
          if (HMAX == 2 && VMAX == 1) { b = (b + (xo & 1)) >> 1; r = (r + (xo & 1)) >> 1; }                      // jcsample.c:226-254
          else if (HMAX == 2 && VMAX == 2) { b = (b + 1 + (xo & 1)) >> 2; r = (r + 1 + (xo & 1)) >> 2; }         // jcsample.c:263-295
          else if (HMAX * VMAX > 1) { b = (b + HMAX * VMAX / 2) / (HMAX * VMAX); r = (r + HMAX * VMAX / 2) / (HMAX * VMAX); }   // jcsample.c:151-190
          cbv[i] = (int16_t)(b - CENTRE); crv[i] = (int16_t)(r - CENTRE);
        }
        int16_t *cb = &sC[rg * CP + seg * (8 / HMAX)], *cr = &sC[8 * CP + rg * CP + seg * (8 / HMAX)];
        if (HMAX == 1) { *reinterpret_cast<uint4 *>(cb) = *reinterpret_cast<const uint4 *>(cbv); *reinterpret_cast<uint4 *>(cr) = *reinterpret_cast<const uint4 *>(crv); }
        else { *reinterpret_cast<uint2 *>(cb) = *reinterpret_cast<const uint2 *>(cbv); *reinterpret_cast<uint2 *>(cr) = *reinterpret_cast<const uint2 *>(crv); }
      }
      };
      if (px4 || pswap) convert(std::true_type{}); else convert(std::false_type{});
    }
    }
  }
  __syncthreads();

  // ---- C: deringing + row pass; 8 lanes per block, lane j owns row j ----
  const int j = tid & 7;
#pragma unroll 1
  for (int b = tid >> 3; b < NB; b += 16) {
    int16_t *plane; int pitch, bx, byl;
    if (b < YB) { plane = sY; pitch = YP; byl = b / YBW; bx = b - byl * YBW; }
    else { int cb = b - YB; int which = cb / CBW; plane = sC + which * 8 * CP; pitch = CP; byl = 0; bx = cb - which * CBW; }
    int16_t *rowp = plane + (byl * 8 + j) * pitch + bx * 8;
    const uint4 rv = *reinterpret_cast<const uint4 *>(rowp);
    int d0 = (int)(int16_t)(rv.x & 0xFFFF), d1 = (int)rv.x >> 16, d2 = (int)(int16_t)(rv.y & 0xFFFF), d3 = (int)rv.y >> 16;
    int d4 = (int)(int16_t)(rv.z & 0xFFFF), d5 = (int)rv.z >> 16, d6 = (int)(int16_t)(rv.w & 0xFFFF), d7 = (int)rv.w >> 16;
    if (DCTM == 2) {
      // convsamp_float -> (float deringing) -> row pass of jpeg_fdct_float; the block's 64 floats sit in sW in natural order
      float f0 = (float)d0, f1 = (float)d1, f2 = (float)d2, f3 = (float)d3, f4 = (float)d4, f5 = (float)d5, f6 = (float)d6, f7 = (float)d7;
      float *w = reinterpret_cast<float *>(sW) + b * 72 + j * 8;
      if (dering) {
        int sum = d0 + d1 + d2 + d3 + d4 + d5 + d6 + d7;          // integer-valued floats add exactly, so the int sum is the float sum
        int cnt = (d0 >= 127) + (d1 >= 127) + (d2 >= 127) + (d3 >= 127) + (d4 >= 127) + (d5 >= 127) + (d6 >= 127) + (d7 >= 127);
        sum += __shfl_xor_sync(0xffffffffu, sum, 1); cnt += __shfl_xor_sync(0xffffffffu, cnt, 1);
        sum += __shfl_xor_sync(0xffffffffu, sum, 2); cnt += __shfl_xor_sync(0xffffffffu, cnt, 2);
        sum += __shfl_xor_sync(0xffffffffu, sum, 4); cnt += __shfl_xor_sync(0xffffffffu, cnt, 4);
        if (cnt != 0 && cnt != 64) {
          w[0] = f0; w[1] = f1; w[2] = f2; w[3] = f3; w[4] = f4; w[5] = f5; w[6] = f6; w[7] = f7;
          __syncwarp(0xFFu << (threadIdx.x & 24));
          if (j == 0) {
            const int ci = b < YB ? 0 : (1 + (b - YB) / CBW);
            deringing_block_float(reinterpret_cast<float *>(sW) + b * 72, (int)qt->q[g.c[ci].qt][0].d >> 3, (float)sum, cnt);
          }
          __syncwarp(0xFFu << (threadIdx.x & 24));
          f0 = w[0]; f1 = w[1]; f2 = w[2]; f3 = w[3]; f4 = w[4]; f5 = w[5]; f6 = w[6]; f7 = w[7];
        }
      }
      fdct_float_1d(f0, f1, f2, f3, f4, f5, f6, f7);
      w[0] = f0; w[1] = f1; w[2] = f2; w[3] = f3; w[4] = f4; w[5] = f5; w[6] = f6; w[7] = f7;
      continue;
    }
    if (dering) {
      int sum = d0 + d1 + d2 + d3 + d4 + d5 + d6 + d7;
      int cnt = (d0 >= 127) + (d1 >= 127) + (d2 >= 127) + (d3 >= 127) + (d4 >= 127) + (d5 >= 127) + (d6 >= 127) + (d7 >= 127);
      sum += __shfl_xor_sync(0xffffffffu, sum, 1); cnt += __shfl_xor_sync(0xffffffffu, cnt, 1);
      sum += __shfl_xor_sync(0xffffffffu, sum, 2); cnt += __shfl_xor_sync(0xffffffffu, cnt, 2);
      sum += __shfl_xor_sync(0xffffffffu, sum, 4); cnt += __shfl_xor_sync(0xffffffffu, cnt, 4);
      if (cnt != 0 && cnt != 64) {
        if (j == 0) {
          const int ci = b < YB ? 0 : (1 + (b - YB) / CBW);
          deringing_block(PlaneAcc{plane + (byl * 8) * pitch + bx * 8, pitch}, (int)qt->q[g.c[ci].qt][0].d >> 3, sum, cnt);
        }
        __syncwarp(0xFFu << (threadIdx.x & 24));          // the 8 lanes of this block
        d0 = rowp[0]; d1 = rowp[1]; d2 = rowp[2]; d3 = rowp[3]; d4 = rowp[4]; d5 = rowp[5]; d6 = rowp[6]; d7 = rowp[7];
      }
    }
    if (DCTM == 1) fdct_ifast_1d(d0, d1, d2, d3, d4, d5, d6, d7);
    else fdct_1d<0, P1>(d0, d1, d2, d3, d4, d5, d6, d7);
    if (DCTM == 2) {
    } else if (PREC == 8) {
      uint4 wv;
      wv.x = ((unsigned)d0 & 0xFFFFu) | ((unsigned)d1 << 16); wv.y = ((unsigned)d2 & 0xFFFFu) | ((unsigned)d3 << 16);
      wv.z = ((unsigned)d4 & 0xFFFFu) | ((unsigned)d5 << 16); wv.w = ((unsigned)d6 & 0xFFFFu) | ((unsigned)d7 << 16);
      *reinterpret_cast<uint4 *>(reinterpret_cast<int16_t *>(sW) + b * 72 + j * 8) = wv;
    } else {
      int *w = reinterpret_cast<int *>(sW) + b * 72 + j * 8;
      w[0] = d0; w[1] = d1; w[2] = d2; w[3] = d3; w[4] = d4; w[5] = d5; w[6] = d6; w[7] = d7;
    }
  }
  __syncthreads();

  // ---- D: column pass + quantize; lane j owns column jc; zigzag placement in the staging buffer.
  //      The four blocks a warp works on own their columns in rotated order (jc), so that their simultaneous 2-byte
  //      stores into the dense 128-byte staging blocks fall into different banks (they were 4-way conflicts).
  //      With the trellis on, the 8 lanes also OR together the zigzag positions of the block's
  //      non-zero plain-quantized AC values for the side record (the trellis kernel finds its
  //      entries from that mask). ----
  int16_t *sQ = reinterpret_cast<int16_t *>(sIO);              // [NB][64] quantized, then [NB][64] raw
  int16_t *sR = sQ + NB * 64;
  static_assert(NB % 16 == 0, "whole warps walk the block list in step");
  const int jc = (j + 2 * ((tid >> 3) & 3)) & 7;
  // zigzag positions of this lane's 8 coefficients (natural index 8r + jc)
  int kz[8];
#pragma unroll
  for (int r = 0; r < 8; r++) {
#if FWD_KZ_PACKED
    kz[r] = (int)((c_izz_col[jc] >> (8 * r)) & 63);
#else
    kz[r] = c_izz[8 * r + jc];
#endif
  }
#pragma unroll 1
  for (int b = tid >> 3; b < NB; b += 16) {
    const wtype *w = sW + b * 72 + jc;
    const int ci = b < YB ? 0 : (1 + (b - YB) / CBW);
    int dd[8], qf[8];                                             // raw coefficients (integers) of this lane's column / float-path quantized values
    if (DCTM == 2) {
      float f0 = w[0], f1 = w[8], f2 = w[16], f3 = w[24], f4 = w[32], f5 = w[40], f6 = w[48], f7 = w[56];
      fdct_float_1d(f0, f1, f2, f3, f4, f5, f6, f7);
      const float ff[8] = {f0, f1, f2, f3, f4, f5, f6, f7};
      const float *fd = qt->fdiv[g.c[ci].qt];
#pragma unroll
      for (int r = 0; r < 8; r++) {
        // forward_DCT_float :860-874 (coefficients for the trellis, as integers; the divisions are in double) ...
        dd[r] = 0;
        if (write_raw) {
          float v = ff[r];
          v = (float)((double)v / c_aan[jc]);                     // i % 8 = column
          v = (float)((double)v / c_aan[r]);                      // i / 8 = row
          dd[r] = (v >= 0.0f) ? (int)((double)v + 0.5) : (int)((double)v - 0.5);
        }
        // ... and quantize_float :808-827
        const float temp = ff[r] * fd[8 * r + jc];
        int q = (int)(int16_t)(__float2int_rz(temp + 16384.5f) - 16384);
        if (dering) q = max(-1023, min(1023, q));
        qf[r] = q;
      }
    } else if (DCTM == 1) {
      int d0 = w[0], d1 = w[8], d2 = w[16], d3 = w[24], d4 = w[32], d5 = w[40], d6 = w[48], d7 = w[56];
      fdct_ifast_1d(d0, d1, d2, d3, d4, d5, d6, d7);
      const int ws8[8] = {d0, d1, d2, d3, d4, d5, d6, d7};
      const IfastConst *ic = qt->ifast[g.c[ci].qt];
#pragma unroll
      for (int r = 0; r < 8; r++) {
        const int nat = 8 * r + jc;
        // raw coefficient for the trellis, rescaled as forward_DCT does (jcdctmgr.c:729-746) ...
        dd[r] = 0;
        if (write_raw) { const int x = ws8[r], sc = c_aanscales[nat]; dd[r] = (x >= 0) ? (x * 32768 + sc) / (2 * sc) : (x * 32768 - sc) / (2 * sc); }
        // ... and the reciprocal quantizer of :611-645 with the scaled divisor's constants (compute_reciprocal :181-230)
        const IfastConst k = ic[nat];
        const int a = abs(ws8[r]);
        int q = (int)(int16_t)(int)(((unsigned long long)(unsigned)(a + (int)k.corr) * k.recip) >> (k.shift + 32));
        if (ws8[r] < 0) q = (int)(int16_t)(-q);
        if (dering) q = max(-1023, min(1023, q));
        qf[r] = q;
      }
    } else {
      int d0 = w[0], d1 = w[8], d2 = w[16], d3 = w[24], d4 = w[32], d5 = w[40], d6 = w[48], d7 = w[56];
      fdct_1d<1, P1>(d0, d1, d2, d3, d4, d5, d6, d7);
      dd[0] = d0; dd[1] = d1; dd[2] = d2; dd[3] = d3; dd[4] = d4; dd[5] = d5; dd[6] = d6; dd[7] = d7;
    }
    const int L = sQL[NC == 1 ? 0 : ci];
    unsigned mlo = 0, mhi = 0;                                 // zigzag positions of this lane's non-zero AC values
#pragma unroll
    for (int r = 0; r < 8; r++) {
      const int nat = 8 * r + jc;
      const int k = kz[r];
      int qv;
      if (DCTM != 0) qv = qf[r];
      else if (QFAST) qv = quant_fast(dd[r], sQC[NC == 1 ? 0 : ci][nat], L, dering);
      else qv = (int)(int16_t)quant_one(dd[r], qt->q[g.c[ci].qt][nat], dering);
      sQ[b * 64 + k] = (int16_t)qv;
      sR[b * 64 + k] = (int16_t)dd[r];
      // the trellis derives its entries from the RAW coefficient (qval = (|x| + q/2) / q, jcdctmgr.c:1136); with the
      // integer DCT that is the plain-quantized value, with the float DCT it can differ from quantize_float's result
      if (!(FWD_MASK_SQ && DCTM == 0)) {
        bool nzv = qv != 0;
        if (DCTM != 0 && rec) { const int dq = (int)qt->q[g.c[ci].qt][nat].d; nzv = abs(dd[r]) >= dq - dq / 2; }
        if (nzv && nat != 0) { if (k < 32) mlo |= 1u << k; else mhi |= 1u << (k - 32); }
      }
    }
    if (PREC == 8 && rec) {
      // the raw coefficients go back to sW in natural order (each lane rewrites exactly the words it read) for
      // phase D2; the 8 lanes OR their non-zero masks together
      if (DCTM == 2) __syncwarp();                             // every lane has read its float column before the int16 view reuses the words
      int16_t *blk16 = reinterpret_cast<int16_t *>(sW + b * 72);     // the block's own words (also when sW holds floats)
      int16_t *ww = blk16 + jc;
#pragma unroll
      for (int r = 0; r < 8; r++) ww[8 * r] = (int16_t)dd[r];
      if (FWD_MASK_SQ && DCTM == 0) {
        // integer DCT: the mask is "which of the block's 64 staged (zigzag-ordered) values are non-zero"; lane j tests
        // the 8 values at positions 8j..8j+7 (two per 32-bit word) and stores its byte of the 64-bit mask
        __syncwarp();
        const uint4 zq = *reinterpret_cast<const uint4 *>(sQ + b * 64 + 8 * j);
        const unsigned zw[4] = {zq.x, zq.y, zq.z, zq.w};
        unsigned m8 = 0;
#pragma unroll
        for (int i = 0; i < 4; i++) {
          const unsigned nz = (((zw[i] & 0x7FFF7FFFu) + 0x7FFF7FFFu) | zw[i]) & 0x80008000u;   // bit 15 / 31: low / high half non-zero
          const unsigned t2 = nz >> 15;
          m8 |= ((t2 | (t2 >> 15)) & 3u) << (2 * i);
        }
        if (j == 0) m8 &= ~1u;                                   // position 0 is the DC value
        reinterpret_cast<uint8_t *>(&sMask[b])[j] = (uint8_t)m8;
      } else {
      mlo |= __shfl_xor_sync(0xffffffffu, mlo, 1); mhi |= __shfl_xor_sync(0xffffffffu, mhi, 1);
      mlo |= __shfl_xor_sync(0xffffffffu, mlo, 2); mhi |= __shfl_xor_sync(0xffffffffu, mhi, 2);
      mlo |= __shfl_xor_sync(0xffffffffu, mlo, 4); mhi |= __shfl_xor_sync(0xffffffffu, mhi, 4);
      if (j == 0) sMask[b] = make_uint2(mlo, mhi);
      }
    }
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // staging writes -> visible to the bulk copies of phase E
  __syncthreads();

  // ---- D2: trellis side records, one thread per block: the serial fp32 sum of squares in NATURAL order
  //      (jcdctmgr.c:1026-1029) over the block's rows (16-byte shared loads; the 144-byte block stride keeps
  //      them conflict-free), the raw DC and the non-zero mask ----
  if (PREC == 8 && rec) {
    for (int b = tid; b < NB; b += 128) {
      int ci, row, col;
      if (b < YB) { ci = 0; int byl = b / YBW; row = ty * VMAX + byl; col = tx * YBW + (b - byl * YBW); }
      else { int cb = b - YB; int which = cb / CBW; ci = 1 + which; row = ty; col = tx * CBW + (cb - which * CBW); }
      const CompGeom &c = g.c[ci];
      if (row >= c.hib || col >= c.wib) continue;
      const int4 *rows = reinterpret_cast<const int4 *>(reinterpret_cast<const int16_t *>(sW + b * 72));
      float norm = 0.0f; int raw_dc = 0;
      // (float)(v * v) without the conversion unit: v as an exact float by the exponent trick, squared in fp32 -- the
      // product of two 16-bit integers rounds to the same float as the converted integer square; the sum itself
      // stays the reference's serial chain
      const float bias = -8421376.0f;   // -(2^23 + 2^15)
#pragma unroll
      for (int r = 0; r < 8; r++) {
        const int4 rv = rows[r];
        const unsigned pw[4] = {(unsigned)rv.x, (unsigned)rv.y, (unsigned)rv.z, (unsigned)rv.w};
#pragma unroll
        for (int cp = 0; cp < 4; cp++) {
          const unsigned u = pw[cp] ^ 0x80008000u;
          float2 f = make_float2(__fadd_rn(__uint_as_float(__byte_perm(u, 0x4B000000u, 0x7610)), bias),
                                 __fadd_rn(__uint_as_float(__byte_perm(u, 0x4B000000u, 0x7632)), bias));
          f.x = __fmul_rn(f.x, f.x); f.y = __fmul_rn(f.y, f.y);
          if (r == 0 && cp == 0) raw_dc = (int)(int16_t)(pw[0] & 0xFFFFu); else norm += f.x;
          norm += f.y;
        }
      }
      const uint2 mk = sMask[b];
      DcRec rr; rr.lambda_dc = norm; rr.raw_dc = (int16_t)raw_dc; rr.nz = (uint8_t)(__popc(mk.x) + __popc(mk.y)); rr.pad = 0;
      rr.nzmask = ((unsigned long long)mk.y << 32) | mk.x;
      const size_t ridx = (size_t)img * rl.per_image + rl.comp_off[ci] + (size_t)row * c.wib + col;
      rec[ridx] = rr;
      // fs.hist: the trellis-phase statistics of the plain-quantized block, encode_mcu_gather's AC half (jchuff.c:886-915,
      // htest_one_block :836-878) walked over the block's non-zero mask -- from sQ itself: with the fast and float DCTs
      // sMask holds the trellis' entries, which come from the raw coefficients -- and its DC value for the DC half
      if (fs.hist) {
        const int16_t *q = sQ + b * 64;
        fs.dcq[ridx] = q[0];
        unsigned long long m;
        if (FWD_MASK_SQ && DCTM == 0) m = rr.nzmask;
        else {
          m = 0;
#pragma unroll
          for (int v = 0; v < 8; v++) {
            const uint4 zq = reinterpret_cast<const uint4 *>(q)[v];
            const unsigned zw[4] = {zq.x, zq.y, zq.z, zq.w};
#pragma unroll
            for (int i = 0; i < 4; i++) {
              const unsigned nz = (((zw[i] & 0x7FFF7FFFu) + 0x7FFF7FFFu) | zw[i]) & 0x80008000u;
              const unsigned t2 = nz >> 15;
              m |= (unsigned long long)((t2 | (t2 >> 15)) & 3u) << (8 * v + 2 * i);
            }
          }
          m &= ~1ull;
        }
        unsigned *h = sHist[NC == 1 ? 0 : ci];
        if (!(m >> 63)) atomicAdd(&h[0], 1u);                  // EOB
        // the mask in two 32-bit halves: a 32-bit lowest-set-bit step is two instructions, the 64-bit one eight
        int prev = 0; unsigned any = 0;
#pragma unroll
        for (int half = 0; half < 2; half++) {
          unsigned w = (unsigned)(m >> (32 * half));
          while (w) {
            const int k = 32 * half + __ffs(w) - 1;
            w &= w - 1;
            const int run = k - prev - 1; prev = k;
            const int a = abs((int)q[k]);
            any |= (unsigned)a;
            if (run >> 4) atomicAdd(&h[0xF0], (unsigned)(run >> 4));
            atomicAdd(&h[((run & 15) << 4) + nbits_of(a)], 1u);  // '+' as walk_seq_block: a 16-bit size lands in bin 256
          }
        }
        // the largest size of the block is the size of the OR of its magnitudes
        if (nbits_of((int)any) > g.max_coef_bits) atomicOr(&fs.status[img], 2u);   // JERR_BAD_DCT_COEF
      }
    }
  }

  // ---- flush (fs.hist): the tile's non-zero AC counts into the image's histograms ----
  if (PREC == 8 && fs.hist) {
    __syncthreads();
    for (int i = tid; i < NC * HW4; i += 128) {              // four bins per thread and step
      const uint4 v = reinterpret_cast<const uint4 *>(&sHist[0][0])[i];
      if ((v.x | v.y | v.z | v.w) == 0) continue;
      const int ci = i / HW4, sym = 4 * (i - ci * HW4);
      unsigned *gh = &fs.hist[(((size_t)img * g.nc + ci) * HIST_SLOTS + 4 + g.c[ci].ac_tbl) * HIST_BINS + sym];
      if (v.x) atomicAdd(gh, v.x);
      if (v.y) atomicAdd(gh + 1, v.y);
      if (v.z) atomicAdd(gh + 2, v.z);
      if (v.w) atomicAdd(gh + 3, v.w);
    }
  }

  // ---- E: whole blocks out.  The blocks of one component's block row inside the tile are consecutive both in the
  //      staging buffer and in the coefficient plane (128 bytes each), so each such run leaves as ONE asynchronous
  //      bulk copy shared -> global (cp.async.bulk, the TMA engine), issued by one thread per run; the threads' own
  //      shared-memory writes were ordered before the async proxy by the fence in front of the barrier above ----
  {
    constexpr int NRUN = VMAX + (NC == 3 ? 2 : 0);
    if (tid < NRUN) {
      int ci, row, col0, b0, maxblk;
      if (tid < VMAX) { ci = 0; row = ty * VMAX + tid; col0 = tx * YBW; b0 = tid * YBW; maxblk = YBW; }
      else { const int which = tid - VMAX; ci = 1 + which; row = ty; col0 = tx * CBW; b0 = YB + which * CBW; maxblk = CBW; }
      const CompGeom &c = g.c[ci];
      const int cnt = row < c.hib ? max(0, min(maxblk, c.wib - col0)) : 0;
      if (cnt > 0) {
        const size_t blk = ((size_t)img * c.hpad + row) * c.wpad + col0;
        const unsigned bytes = (unsigned)cnt * 128u;
        if (!fs.hist)                                            // with the statistics counted here nobody reads the plain plane
          asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                       :: "l"(c.coef + blk * 64), "r"((unsigned)__cvta_generic_to_shared(sQ + b0 * 64)), "r"(bytes) : "memory");
        if (write_raw)                                           // only the trellis (and the debug tap) read the raw DCT
          asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                       :: "l"(c.raw + blk * 64), "r"((unsigned)__cvta_generic_to_shared(sR + b0 * 64)), "r"(bytes) : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");    // the staging buffer must outlive the reads
      }
    }
  }
}

// cuTensorMapEncodeTiled through the runtime's driver entry point query (no link against libcuda)
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
                                  const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn tensor_map_encoder()
{
  static EncodeTiledFn fn = [] {
    void *p = nullptr; cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) p = nullptr;
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}
// The batch's pixels as a rank-3 byte tensor {W * samples per pixel, H, n}; box = one tile (or half of one) of the
// forward kernel.  Returns 0 when the layout does not qualify (alignment, pixel order, sample size): the kernel
// then loads with ordinary global loads.  A zero image stride (every image reads the same pixels) maps one image,
// which the kernel addresses as image 0.
static int make_pixel_tensor_map(const Geom &g, const uint8_t *src, int n, int ic, int tile_rows, CUtensorMap *tm)
{
  static const bool off = getenv("B200JPEG_NO_TMA") != nullptr;     // A/B aid
  memset(tm, 0, sizeof *tm);
  EncodeTiledFn enc = tensor_map_encoder();
  if (off || !enc || g.raw_in || !src || g.in_comps != ic || g.px_swap || g.px_first || g.max_coef_bits != 10) return 0;
  if (g.image_stride == 0) n = 1;
  if (((size_t)src & 15) || (g.row_pitch & 15) || (n > 1 && (g.image_stride & 15))) return 0;
  const cuuint64_t dims[3] = {(cuuint64_t)g.W * ic, (cuuint64_t)g.H, (cuuint64_t)n};
  const cuuint64_t strides[2] = {(cuuint64_t)g.row_pitch, (cuuint64_t)(n > 1 ? g.image_stride : ((g.row_pitch * (size_t)g.H + 15) & ~(size_t)15))};
  const cuuint32_t box[3] = {(cuuint32_t)(ic == 3 ? 192 : 128), (cuuint32_t)tile_rows, 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  return enc(tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<uint8_t *>(src), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <bool QFAST, int PREC, int DCTM>
static void launch_forward_tile(const Geom &g, const uint8_t *src, const QuantTables *qt, int dering, DcRec *rec, const RecLayout &rl, const FwdStats &fs, int n, cudaStream_t s, bool gray, int write_raw)
{
  dim3 grid((g.W + 127) / 128, g.mcu_rows, n);
  CUtensorMap tm;
  const int use_tma = PREC == 8 ? make_pixel_tensor_map(g, src, n, gray ? 1 : 3, 8 * (gray ? 1 : g.vmax), &tm) : (memset(&tm, 0, sizeof tm), 0);
  if (gray) k_forward_tile<1, 1, 1, QFAST, PREC, DCTM><<<grid, 128, 0, s>>>(g, src, qt, dering, rec, rl, write_raw, fs, tm, use_tma);
  else if (g.hmax == 1 && g.vmax == 1) k_forward_tile<1, 1, 3, QFAST, PREC, DCTM><<<grid, 128, 0, s>>>(g, src, qt, dering, rec, rl, write_raw, fs, tm, use_tma);
  else if (g.hmax == 2 && g.vmax == 1) k_forward_tile<2, 1, 3, QFAST, PREC, DCTM><<<grid, 128, 0, s>>>(g, src, qt, dering, rec, rl, write_raw, fs, tm, use_tma);
  else if (g.hmax == 1 && g.vmax == 2) k_forward_tile<1, 2, 3, QFAST, PREC, DCTM><<<grid, 128, 0, s>>>(g, src, qt, dering, rec, rl, write_raw, fs, tm, use_tma);
  else k_forward_tile<2, 2, 3, QFAST, PREC, DCTM><<<grid, 128, 0, s>>>(g, src, qt, dering, rec, rl, write_raw, fs, tm, use_tma);
}
// =====================================================================
// Input smoothing (cinfo->smoothing_factor, cjpeg -smooth N).  The smoothing downsamplers (jcsample.c:298-455) read a
// row and a column of context around every sample, and the pre-processing controller then runs in context mode
// (pre_process_context, jcprepct.c:201-262), which also changes how rows past the image bottom come about: every
// output row is downsampled from input rows clamped to the last one (not replicated after downsampling).  That case
// runs as its own pre-pass: colour conversion + the methods jinit_downsampler picks (jcsample.c:463-545) into component
// planes of hib*8 x wib*8 samples, which the forward kernel then takes like raw-data input.
//   full-size component : fullsize_smooth_downsample  (member*(65536 - 512 SF) + 8 neighbours * 64 SF)
//   2h x 2v             : h2v2_smooth_downsample      (4 members * (16384 - 80 SF) + (2 * 8 edge + 4 corner neighbours) * 16 SF)
//   anything else       : the plain box filters (h2v1 bias 0,1,..; int_downsample rounded mean) - no smoothing there
// Edge columns: the reference's first/last-column special cases equal clamping the column index to [0, W-1].
// =====================================================================
template <int SB>
__global__ void __launch_bounds__(128) k_prep_planes(Geom g, const uint8_t *__restrict__ src, int sf, PlanesOut out)
{
  const int ci = blockIdx.z % g.nc, img = blockIdx.z / g.nc;
  const CompGeom &c = g.c[ci];
  const int xo = blockIdx.x * blockDim.x + threadIdx.x, yo = blockIdx.y;
  if (xo >= c.wib * 8 || yo >= c.hib * 8) return;
  const uint8_t *base = src + (size_t)img * g.image_stride;
  const int comp = g.cs_mode == 1 ? 0 : ci;
  auto at = [&](int y, int x) -> int {
    y = max(0, min(y, g.H - 1)); x = max(0, min(x, g.W - 1));
    return convert_sample<SB>(base + (size_t)y * g.row_pitch + (size_t)x * g.in_comps * SB, g.cs_mode, comp, g.px_first, g.px_swap);
  };
  int val;
  if (c.hx == 1 && c.vx == 1) {
    const int member = at(yo, xo);
    int neigh = -member;
    for (int dy = -1; dy <= 1; dy++) for (int dx = -1; dx <= 1; dx++) neigh += at(yo + dy, xo + dx);
    val = (member * (65536 - sf * 512) + neigh * (sf * 64) + 32768) >> 16;
  } else if (c.hx == 2 && c.vx == 2) {
    const int y = 2 * yo, x = 2 * xo;
    const int member = at(y, x) + at(y, x + 1) + at(y + 1, x) + at(y + 1, x + 1);
    int edge = at(y - 1, x) + at(y - 1, x + 1) + at(y + 2, x) + at(y + 2, x + 1) + at(y, x - 1) + at(y, x + 2) + at(y + 1, x - 1) + at(y + 1, x + 2);
    const int corner = at(y - 1, x - 1) + at(y - 1, x + 2) + at(y + 2, x - 1) + at(y + 2, x + 2);
    val = (member * (16384 - sf * 80) + (2 * edge + corner) * (sf * 16) + 32768) >> 16;
  } else {
    int sum = 0;
    for (int dv = 0; dv < c.vx; dv++) for (int du = 0; du < c.hx; du++) sum += at(yo * c.vx + dv, xo * c.hx + du);
    if (c.hx == 2 && c.vx == 1) val = (sum + (xo & 1)) >> 1;
    else { const int np = c.hx * c.vx; val = (sum + np / 2) / np; }
  }
  uint8_t *dst = out.p[ci] + (size_t)img * out.stride[ci] + (size_t)yo * out.pitch[ci] + (size_t)xo * SB;
  if (SB == 1) *dst = (uint8_t)val; else *reinterpret_cast<uint16_t *>(dst) = (uint16_t)val;
}
void launch_prep_planes(const Geom &g, const uint8_t *src, int smoothing_factor, const PlanesOut &out, int n, cudaStream_t s)
{
  int mw = 0, mh = 0;
  for (int ci = 0; ci < g.nc; ci++) { mw = max(mw, g.c[ci].wib * 8); mh = max(mh, g.c[ci].hib * 8); }
  dim3 grid((mw + 127) / 128, mh, n * g.nc);
  if (g.max_coef_bits == 14) k_prep_planes<2><<<grid, 128, 0, s>>>(g, src, smoothing_factor, out);
  else k_prep_planes<1><<<grid, 128, 0, s>>>(g, src, smoothing_factor, out);
  LAUNCHED();
}

// =====================================================================
// TurboJPEG YUV planes (tj3EncodeYUVPlanes8, turbojpeg.c:1467-1619): colour conversion + the downsamplers
// jinit_downsampler picks without smoothing (jcsample.c:463-545), written straight into the caller's planes.
// One CTA = one tile of YUV_TH rows x YUV_TW pixels of one image:
//   A. the tile's input rows are read once, with 16-byte loads at 16-byte aligned addresses (byte loads at the ragged
//      ends), into shared memory at the source's 16-byte phase; rows past the image are the last row (turbojpeg.c:
//      1539-1540), columns past it the last column (expand_right_edge, jcsample.c:98-116);
//   B. every pixel is converted once (convert_sample) and its luma sample stored, and each HX x VX group of pixels sums
//      into one sample per chroma plane: h2v1_downsample (bias 0,1,..), h2v2_downsample (bias 1,2,..), int_downsample
//      (rounded mean) for the other ratios; the output rows are staged at the destination's 16-byte phase;
//   C. every plane row segment is written with 16-byte stores, byte stores only at its two ends, so bytes of the
//      caller's pitch padding past pw[ci] are never touched.
// The layout the kernel covers is every TJSAMP_*: component 0 at the maximum sampling factors (HX = hmax, VX = vmax),
// components 1 and 2 (if any) 1x1.
// =====================================================================
#define YUV_TW 256
#define YUV_TH 16
template <int HX, int VX, int PS>
__global__ void __launch_bounds__(256) k_encode_yuv(Geom g, const uint8_t *__restrict__ src, YuvOut out)
{
  constexpr int CW = YUV_TW / HX, CH = YUV_TH / VX;
  __shared__ __align__(16) uint8_t s_in[YUV_TH][YUV_TW * PS + 16];
  __shared__ __align__(16) uint8_t s_y[YUV_TH][YUV_TW + 16];
  __shared__ __align__(16) uint8_t s_c[2][CH][CW + 16];
  __shared__ int s_head[YUV_TH], s_hy[YUV_TH], s_hc[2][CH];
  const int img = blockIdx.z, x0 = blockIdx.x * YUV_TW, y0 = blockIdx.y * YUV_TH;
  const int ncols = min(YUV_TW, g.W - x0);              // >= 1: YUV_TW is a multiple of hmax, so no tile starts in pw0's padding
  const int ow = min(YUV_TW, out.pw[0] - x0);           // luma columns of this tile inside the plane
  const uint8_t *base = src + (size_t)img * g.image_stride;
  auto plane_row = [&](int ci, int y) { return out.p[ci] + (size_t)img * out.stride[ci] + (size_t)y * out.pitch[ci] + x0 / (ci ? HX : 1); };
  if (threadIdx.x < YUV_TH) {
    const int r = threadIdx.x;
    s_head[r] = (int)((uintptr_t)(base + (size_t)min(y0 + r, g.H - 1) * g.row_pitch + (size_t)x0 * PS) & 15);
    s_hy[r] = (int)((uintptr_t)plane_row(0, y0 + r) & 15);
    if (r < CH && g.nc == 3) { s_hc[0][r] = (int)((uintptr_t)plane_row(1, y0 / VX + r) & 15); s_hc[1][r] = (int)((uintptr_t)plane_row(2, y0 / VX + r) & 15); }
  }
  __syncthreads();
  // A. load
  {
    const int nbytes = ncols * PS, words = (YUV_TW * PS + 16) / 16;
    for (int i = threadIdx.x; i < YUV_TH * words; i += blockDim.x) {
      const int r = i / words, w = i - r * words, head = s_head[r];
      const int b0 = 16 * w - head;                      // first byte of the word, relative to the row's first byte
      if (b0 >= nbytes) continue;
      const uint8_t *row = base + (size_t)min(y0 + r, g.H - 1) * g.row_pitch + (size_t)x0 * PS;
      if (b0 >= 0 && b0 + 16 <= nbytes) {
        *reinterpret_cast<uint4 *>(&s_in[r][16 * w]) = __ldg(reinterpret_cast<const uint4 *>(row + b0));
      } else {
        for (int b = max(b0, 0); b < min(b0 + 16, nbytes); b++) s_in[r][head + b] = __ldg(row + b);
      }
    }
  }
  __syncthreads();
  // B. convert + downsample
  for (int i = threadIdx.x; i < CH * CW; i += blockDim.x) {
    const int gr = i / CW, gc = i - gr * CW;
    int sum1 = 0, sum2 = 0;
#pragma unroll
    for (int dv = 0; dv < VX; dv++) {
      const int r = gr * VX + dv;
#pragma unroll
      for (int du = 0; du < HX; du++) {
        const int x = gc * HX + du;
        const uint8_t *px = &s_in[r][s_head[r] + min(x, ncols - 1) * PS];
        s_y[r][s_hy[r] + x] = (uint8_t)convert_sample<1>(px, g.cs_mode, 0, g.px_first, g.px_swap);
        if (g.nc == 3) { sum1 += convert_sample<1>(px, g.cs_mode, 1, g.px_first, g.px_swap); sum2 += convert_sample<1>(px, g.cs_mode, 2, g.px_first, g.px_swap); }
      }
    }
    if (g.nc == 3) {
      int v1, v2;
      if (HX == 1 && VX == 1) { v1 = sum1; v2 = sum2; }
      else if (HX == 2 && VX == 1) { const int bias = gc & 1; v1 = (sum1 + bias) >> 1; v2 = (sum2 + bias) >> 1; }          // x0 is even
      else if (HX == 2 && VX == 2) { const int bias = 1 + (gc & 1); v1 = (sum1 + bias) >> 2; v2 = (sum2 + bias) >> 2; }
      else { constexpr int NP = HX * VX; v1 = (sum1 + NP / 2) / NP; v2 = (sum2 + NP / 2) / NP; }
      s_c[0][gr][s_hc[0][gr] + gc] = (uint8_t)v1; s_c[1][gr][s_hc[1][gr] + gc] = (uint8_t)v2;
    }
  }
  __syncthreads();
  // C. store: plane 0 (YUV_TH rows of ow samples), then planes 1, 2 (CH rows of ow / HX samples)
  const int nplanes = g.nc == 3 ? 3 : 1;
  for (int ci = 0; ci < nplanes; ci++) {
    const int rows = ci ? CH : YUV_TH, cols = ci ? ow / HX : ow, ry0 = ci ? y0 / VX : y0;
    const int words = ((ci ? CW : YUV_TW) + 16) / 16;
    for (int i = threadIdx.x; i < rows * words; i += blockDim.x) {
      const int r = i / words, w = i - r * words;
      if (ry0 + r >= out.ph[ci]) continue;
      const int head = ci ? s_hc[ci - 1][r] : s_hy[r];
      const uint8_t *srow = ci ? &s_c[ci - 1][r][0] : &s_y[r][0];
      const int b0 = 16 * w - head;
      if (b0 >= cols) continue;
      uint8_t *drow = plane_row(ci, ry0 + r);
      if (b0 >= 0 && b0 + 16 <= cols) *reinterpret_cast<uint4 *>(drow + b0) = *reinterpret_cast<const uint4 *>(srow + 16 * w);
      else for (int b = max(b0, 0); b < min(b0 + 16, cols); b++) drow[b] = srow[head + b];
    }
  }
}
template <int HX, int VX>
static void launch_encode_yuv_hv(const Geom &g, const uint8_t *src, const YuvOut &out, dim3 grid, cudaStream_t s)
{
  if (g.in_comps == 1) k_encode_yuv<HX, VX, 1><<<grid, 256, 0, s>>>(g, src, out);
  else if (g.in_comps == 3) k_encode_yuv<HX, VX, 3><<<grid, 256, 0, s>>>(g, src, out);
  else k_encode_yuv<HX, VX, 4><<<grid, 256, 0, s>>>(g, src, out);
}
void launch_encode_yuv(const Geom &g, const uint8_t *src, const YuvOut &out, int n, cudaStream_t s)
{
  const dim3 grid((out.pw[0] + YUV_TW - 1) / YUV_TW, (out.ph[0] + YUV_TH - 1) / YUV_TH, n);
  switch (g.hmax * 8 + g.vmax) {
  case 9:  launch_encode_yuv_hv<1, 1>(g, src, out, grid, s); break;
  case 10: launch_encode_yuv_hv<1, 2>(g, src, out, grid, s); break;
  case 12: launch_encode_yuv_hv<1, 4>(g, src, out, grid, s); break;
  case 17: launch_encode_yuv_hv<2, 1>(g, src, out, grid, s); break;
  case 18: launch_encode_yuv_hv<2, 2>(g, src, out, grid, s); break;
  case 20: launch_encode_yuv_hv<2, 4>(g, src, out, grid, s); break;
  case 33: launch_encode_yuv_hv<4, 1>(g, src, out, grid, s); break;
  case 34: launch_encode_yuv_hv<4, 2>(g, src, out, grid, s); break;
  default: launch_encode_yuv_hv<4, 4>(g, src, out, grid, s); break;
  }
  LAUNCHED();
}

// fast path: full-size first component, (for colour) two 1x1-sampled chroma components
static bool forward_gray(const Geom &g) { return g.nc == 1 && (g.raw_in || g.cs_mode == 1 || (g.cs_mode == 2 && g.in_comps == 1)); }
bool forward_tiled(const Geom &g, int dct_method)
{
  const bool ycc = g.nc == 3 && (g.raw_in || (g.cs_mode == 0 && (g.in_comps == 3 || g.in_comps == 4))) && g.c[0].h == g.hmax && g.c[0].v == g.vmax &&
                   g.c[1].h == 1 && g.c[1].v == 1 && g.c[2].h == 1 && g.c[2].v == 1 && g.hmax <= 2 && g.vmax <= 2;
  static const bool force_generic = getenv("B200JPEG_GENERIC_FORWARD") != nullptr;   // A/B switch for debugging
  // (12-bit samples with the fast / float DCT: the one-thread-per-block kernel only)
  return !force_generic && ((forward_gray(g) && g.hmax == 1 && g.vmax == 1) || ycc) && !(g.max_coef_bits == 14 && dct_method != 0);
}
void launch_forward(const Geom &g, const uint8_t *src, const QuantTables *qt, int qfast, int dct_method, int dering, DcRec *rec, const RecLayout &rl, int keep_raw,
                    const FwdStats &fs, int n, cudaStream_t s)
{
  const int write_raw = rec != nullptr || keep_raw;
  const bool gray = forward_gray(g);
  if (forward_tiled(g, dct_method)) {
    const FwdStats none = {nullptr, nullptr, nullptr};
    if (g.max_coef_bits == 14) {                       // 12-bit samples (uint16)
      if (qfast) launch_forward_tile<true, 12, 0>(g, src, qt, 0, nullptr, rl, none, n, s, gray, 0);
      else launch_forward_tile<false, 12, 0>(g, src, qt, 0, nullptr, rl, none, n, s, gray, 0);
    } else if (dct_method == 2) launch_forward_tile<true, 8, 2>(g, src, qt, dering, rec, rl, fs, n, s, gray, write_raw);
    else if (dct_method == 1) launch_forward_tile<true, 8, 1>(g, src, qt, dering, rec, rl, fs, n, s, gray, write_raw);
    else if (qfast) launch_forward_tile<true, 8, 0>(g, src, qt, dering, rec, rl, fs, n, s, gray, write_raw);
    else launch_forward_tile<false, 8, 0>(g, src, qt, dering, rec, rl, fs, n, s, gray, write_raw);
    LAUNCHED();
    return;
  }
  // every other sampling layout (3x2, 4x1, luma-subsampled, RGB pass-through, ...): one thread per block
  int mw = 0, mh = 0;
  for (int ci = 0; ci < g.nc; ci++) { mw = max(mw, g.c[ci].wib); mh = max(mh, g.c[ci].hib); }
  dim3 grid((mw + 127) / 128, mh, n * g.nc);
  if (g.max_coef_bits == 14) {
    if (dct_method == 2) k_forward<12, 2><<<grid, 128, 0, s>>>(g, src, qt, 0, nullptr, rl);
    else if (dct_method == 1) k_forward<12, 1><<<grid, 128, 0, s>>>(g, src, qt, 0, nullptr, rl);
    else k_forward<12, 0><<<grid, 128, 0, s>>>(g, src, qt, 0, nullptr, rl);
  }
  else if (dct_method == 2) k_forward<8, 2><<<grid, 128, 0, s>>>(g, src, qt, dering, rec, rl);
  else if (dct_method == 1) k_forward<8, 1><<<grid, 128, 0, s>>>(g, src, qt, dering, rec, rl);
  else k_forward<8, 0><<<grid, 128, 0, s>>>(g, src, qt, dering, rec, rl);
  LAUNCHED();
}

// =====================================================================
// Coefficient-domain input (jpeg_write_coefficients, jctrans.c:39-66 / compress_output :303-378): the caller's
// blocks are libjpeg JBLOCKs (natural order, width_in_blocks x height_in_blocks per component); they go into the
// padded zigzag-order planes every later stage reads.  Dummy blocks are made by k_dummy as on the pixel path: the
// transcoder's rule (DC of the previous block of the MCU, jctrans.c:352-362) gives the same values.
// A lossless transform (jpegtran's do_* routines, transupp.c:727-1357) is this copy's gather: the destination block
// picks its source block by the CoefXform mapping and its coefficients through one of eight in-block operations.
// =====================================================================
// in-block operation op = transposed * 4 + (x axis mirrored) * 2 + (y axis mirrored): for destination zigzag position
// k, the natural source index | 0x100 when the value is negated (a mirrored axis negates its odd frequencies).  Kept in
// global memory and read through L1: a warp's 32 lanes read 32 different entries, which __constant__ memory would
// serialise.
struct XfTab { unsigned short e[8][64]; };
constexpr XfTab make_xf_tab()
{
  constexpr unsigned char zz[64] = {0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
                                    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
  XfTab t{};
  for (int op = 0; op < 8; op++)
    for (int k = 0; k < 64; k++) {
      const int n = zz[k], r = n >> 3, c = n & 7;
      const int neg = (((op >> 1) & 1) & c) ^ ((op & 1) & r);
      t.e[op][k] = (unsigned short)(((op & 4) ? c * 8 + r : n) | (neg << 8));
    }
  return t;
}
__device__ const XfTab g_xf = make_xf_tab();

__global__ void __launch_bounds__(256) k_import_coefs(Geom g, const __grid_constant__ CoefXform xf)
{
  const int ci = blockIdx.y % g.nc, img = blockIdx.y / g.nc;
  const CompGeom &c = g.c[ci];
  const long long nblk = (long long)c.wib * c.hib;
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;     // (block, zigzag position)
  if (t >= nblk * 64) return;
  const long long b = t >> 6; const int k = (int)(t & 63);
  const int row = (int)(b / c.wib), col = (int)(b - (long long)row * c.wib);
  int ax = col + xf.x_crop[ci], ay = row + xf.y_crop[ci];
  const int xm = ax < xf.x_mirror[ci], ym = ay < xf.y_mirror[ci];
  if (xm) ax = xf.x_mirror[ci] - 1 - ax;
  if (ym) ay = xf.y_mirror[ci] - 1 - ay;
  const int sr = xf.transposed ? ax : ay, sc = xf.transposed ? ay : ax;
  const int e = __ldg(&g_xf.e[xf.transposed * 4 + xm * 2 + ym][k]);
  const int16_t *src = reinterpret_cast<const int16_t *>(g.plane[ci] + (size_t)img * g.plane_stride[ci] + (size_t)sr * g.plane_pitch[ci]) + (size_t)sc * 64;
  const int16_t v = src[e & 63];
  c.coef[(((size_t)img * c.hpad + row) * c.wpad + col) * 64 + k] = (e & 0x100) ? (int16_t)-v : v;
}
void launch_import_coefs(const Geom &g, const CoefXform &xf, int n, cudaStream_t s)
{
  long long mb = 0;
  for (int ci = 0; ci < g.nc; ci++) mb = max(mb, (long long)g.c[ci].wib * g.c[ci].hib);
  dim3 grid((unsigned)((mb * 64 + 255) / 256), n * g.nc);
  k_import_coefs<<<grid, 256, 0, s>>>(g, xf);
  LAUNCHED();
}

// =====================================================================
// dummy blocks (jccoefct.c:312-345 == :443-476): AC = 0; right-edge dummies
// take the DC of the last real block of the row, bottom dummy rows take, per
// MCU, the DC of the last block of that MCU in the row above.
// =====================================================================
__global__ void k_dummy(Geom g)
{
  const int ci = blockIdx.y % g.nc, img = blockIdx.y / g.nc;
  const CompGeom &c = g.c[ci];
  long long nd_right = (long long)c.hib * (c.wpad - c.wib);
  long long nd = nd_right + (long long)(c.hpad - c.hib) * c.wpad;
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nd) return;
  int r, b, srow, scol;
  if (t < nd_right) { r = (int)(t / (c.wpad - c.wib)); b = c.wib + (int)(t % (c.wpad - c.wib)); srow = r; scol = c.wib - 1; }
  else {
    long long u = t - nd_right; r = c.hib + (int)(u / c.wpad); b = (int)(u % c.wpad);
    srow = c.hib - 1; scol = min((b / c.h) * c.h + c.h - 1, c.wib - 1);
  }
  int16_t *dst = c.coef + (((size_t)img * c.hpad + r) * c.wpad + b) * 64;
  int16_t dc = c.coef[(((size_t)img * c.hpad + srow) * c.wpad + scol) * 64];
  uint4 *d4 = reinterpret_cast<uint4 *>(dst);
  d4[0] = make_uint4((unsigned)(uint16_t)dc, 0, 0, 0);
  for (int v = 1; v < 8; v++) d4[v] = make_uint4(0, 0, 0, 0);
}
void launch_dummy(const Geom &g, int n, cudaStream_t s)
{
  long long nd = 0;
  for (int ci = 0; ci < g.nc; ci++) { const CompGeom &c = g.c[ci]; nd = max(nd, (long long)c.hib * (c.wpad - c.wib) + (long long)(c.hpad - c.hib) * c.wpad); }
  if (nd == 0) return;
  dim3 grid((unsigned)((nd + 127) / 128), n * g.nc);
  k_dummy<<<grid, 128, 0, s>>>(g);
  LAUNCHED();
}

// =====================================================================
// scan-order block addressing (compress_output, jccoefct.c:498-553)
// =====================================================================
struct BlockRef { const int16_t *blk; int sci; int mcu; int k; };

__device__ __forceinline__ const int16_t *block_ptr(const Geom &g, const ScanDesc &sd, int img, long long t, int &sci, long long &mcu, int &k)
{
  mcu = t / sd.bim; k = (int)(t - mcu * sd.bim);
  sci = sd.k_comp[k];
  const CompGeom &c = g.c[sd.ci[sci]];
  long long mrow = mcu / sd.per_row; int mcol = (int)(mcu - mrow * sd.per_row);
  int mh = sd.ncomps == 1 ? 1 : c.v, mw = sd.ncomps == 1 ? 1 : c.h;
  long long row = mrow * mh + sd.k_y[k]; int col = mcol * mw + sd.k_x[k];
  return c.coef + (((size_t)img * c.hpad + row) * c.wpad + col) * 64;
}
// DC value of the previous block of the same component in scan order (or 0)
__device__ __forceinline__ int prev_dc(const Geom &g, const ScanDesc &sd, int img, long long t, int sci, long long mcu, int k)
{
  long long tp;
  if (k > sd.k_first[sci]) tp = t - 1;
  else if (mcu > 0 && !(sd.ri && mcu % sd.ri == 0)) tp = t - sd.bim + sd.k_count[sci] - 1;   // emit_restart resets last_dc_val (jchuff.c:681-683)
  else return 0;
  int s2, k2; long long m2;
  const int16_t *p = block_ptr(g, sd, img, tp, s2, m2, k2);
  return p[0];
}

// Walks one block the way encode_one_block (jchuff.c:563-661) / htest_one_block
// (jchuff.c:812-878) do, calling sink.dc(nbits, valuebits) and
// sink.ac(symbol, nbits, valuebits) in stream order.
// ld(v): the block's v-th group of 8 zigzag-ordered coefficients (16 bytes)
template <class Sink, class Load>
__device__ __forceinline__ void walk_seq_chunks(Load ld, int last_dc, Sink &sink)
{
  int r = 0;
#pragma unroll
  for (int v = 0; v < 8; v++) {
    uint4 q = ld(v);
    unsigned w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int j = 0; j < 8; j++) {
      int val = (int)(int16_t)((w[j >> 1] >> ((j & 1) * 16)) & 0xFFFF);
      if (v == 0 && j == 0) {
        int temp = val - last_dc, temp2 = temp;
        if (temp < 0) { temp = -temp; temp2--; }
        int nb = nbits_of(temp);
        sink.dc(nb, temp2);
      } else if (val == 0) {
        r++;
      } else {
        while (r > 15) { sink.ac(0xF0, 0, 0); r -= 16; }
        int temp = val, temp2 = val;
        if (temp < 0) { temp = -temp; temp2--; }
        int nb = nbits_of(temp);
        sink.ac((r << 4) + nb, nb, temp2);
        r = 0;
      }
    }
  }
  if (r > 0) sink.ac(0, 0, 0);
}
template <class Sink>
__device__ __forceinline__ void walk_seq_block(const int16_t *__restrict__ blk, int last_dc, Sink &sink)
{
  const uint4 *b4 = reinterpret_cast<const uint4 *>(blk);
  walk_seq_chunks([&](int v) { return b4[v]; }, last_dc, sink);
}

#ifndef SEQ_SPARSE_ENC
#define SEQ_SPARSE_ENC 1
#endif
// the same sparse walk in the statistics and bit-count kernels: measured slower than the dense 16-byte loads there
// (0.61 / 0.62 vs 0.53 / 0.57 ms per 64 4K images), so off
#ifndef SEQ_SPARSE_STATS
#define SEQ_SPARSE_STATS 0
#endif
// Zigzag positions of a scan-order block's non-zero AC coefficients, from the side records (the AC trellis leaves the
// final ones there); dummy blocks have none.
__device__ __forceinline__ unsigned long long block_nzmask(const Geom &g, const ScanDesc &sd, const DcRec *__restrict__ rec, const RecLayout &rl,
                                                           int img, int sci, long long mcu, int k)
{
  const int ci = sd.ci[sci];
  const CompGeom &c = g.c[ci];
  const long long mrow = mcu / sd.per_row; const int mcol = (int)(mcu - mrow * sd.per_row);
  const int mh = sd.ncomps == 1 ? 1 : c.v, mw = sd.ncomps == 1 ? 1 : c.h;
  const long long row = mrow * mh + sd.k_y[k]; const int col = mcol * mw + sd.k_x[k];
  return (row < c.hib && col < c.wib) ? rec[(size_t)img * rl.per_image + rl.comp_off[ci] + (size_t)row * c.wib + col].nzmask : 0ull;
}
// walk_seq_block for a block whose non-zero positions are known: touches only those coefficients
template <class Sink>
__device__ __forceinline__ void walk_seq_sparse(const int16_t *__restrict__ blk, unsigned long long mask, int last_dc, Sink &sink)
{
  if (mask & 0xFFFF0000ull) asm volatile("prefetch.global.L1 [%0];" :: "l"(blk + 16));
  if (mask & 0xFFFF00000000ull) asm volatile("prefetch.global.L1 [%0];" :: "l"(blk + 32));
  if (mask >> 48) asm volatile("prefetch.global.L1 [%0];" :: "l"(blk + 48));
  {
    int temp = (int)blk[0] - last_dc, temp2 = temp;
    if (temp < 0) { temp = -temp; temp2--; }
    sink.dc(nbits_of(temp), temp2);
  }
  int prev = 0;
  while (mask) {
    const int pos = __ffsll((long long)mask) - 1;
    mask &= mask - 1;
    const int val = blk[pos];
    if (val == 0) continue;                              // a superset mask is fine
    int r = pos - prev - 1; prev = pos;
    while (r > 15) { sink.ac(0xF0, 0, 0); r -= 16; }
    int temp = val, temp2 = val;
    if (temp < 0) { temp = -temp; temp2--; }
    const int nb = nbits_of(temp);
    sink.ac((r << 4) + nb, nb, temp2);
  }
  if (prev != 63) sink.ac(0, 0, 0);
}


// ---------------------------------------------------------------------
// Sequential scans after the AC trellis: the blocks' symbols come from the records the trellis back-track left (SymOut,
// kernels.cuh) and the DC values from the dense array the DC trellis wrote -- the 128-byte coefficient blocks are not read.
// ---------------------------------------------------------------------
// scan-order block -> block coordinates inside its component (compress_output, jccoefct.c:498-553).  A scan has fewer
// than 2^31 blocks (65500 x 65500 samples at most), so the arithmetic is 32-bit.
struct ScanPos { int sci, k, mrow, mcol, row, col; unsigned mcu; };
__device__ __forceinline__ void scan_place(const Geom &g, const ScanDesc &sd, ScanPos &p)
{
  const CompGeom &c = g.c[sd.ci[p.sci]];
  const int mh = sd.ncomps == 1 ? 1 : c.v, mw = sd.ncomps == 1 ? 1 : c.h;
  p.row = p.mrow * mh + sd.k_y[p.k]; p.col = p.mcol * mw + sd.k_x[p.k];
}
__device__ __forceinline__ ScanPos scan_coords(const Geom &g, const ScanDesc &sd, long long t)
{
  ScanPos p;
  const unsigned tt = (unsigned)t, bim = (unsigned)sd.bim, per_row = (unsigned)sd.per_row;
  p.mcu = bim == 1 ? tt : tt / bim; p.k = (int)(tt - p.mcu * bim);
  p.sci = sd.k_comp[p.k];
  p.mrow = (int)(p.mcu / per_row); p.mcol = (int)(p.mcu - (unsigned)p.mrow * per_row);
  scan_place(g, sd, p);
  return p;
}
// final DC value of the block at (row, col) of a component; d = the image's dense DC values of that component.  Dummy
// blocks repeat a real block's value, the one k_dummy copies (jccoefct.c:312-345, :443-476)
__device__ __forceinline__ int dense_dc(const CompGeom &c, const int16_t *__restrict__ d, int row, int col)
{
  if (row >= c.hib) { row = c.hib - 1; col = min(c.h == 1 ? col : (col / c.h) * c.h + c.h - 1, c.wib - 1); }
  else if (col >= c.wib) col = c.wib - 1;
  return d[(size_t)row * c.wib + col];
}
// DC value of the previous block of the same component in scan order (0 at the scan's start and after a restart marker):
// the block before it in the same MCU, or the component's last block of the MCU before
__device__ __forceinline__ int prev_dc_dense(const Geom &g, const ScanDesc &sd, const int16_t *__restrict__ dimg /* the image's dense DC values */,
                                             const RecLayout &rl, const ScanPos &p)
{
  ScanPos q = p;
  if (p.k > sd.k_first[p.sci]) q.k = p.k - 1;
  else if (p.mcu > 0 && !(sd.ri && p.mcu % (unsigned)sd.ri == 0)) {                            // emit_restart resets last_dc_val (jchuff.c:681-683)
    q.k = sd.k_first[p.sci] + sd.k_count[p.sci] - 1;
    if (p.mcol > 0) q.mcol = p.mcol - 1; else { q.mrow = p.mrow - 1; q.mcol = sd.per_row - 1; }
  } else return 0;
  scan_place(g, sd, q);
  const int ci = sd.ci[p.sci];
  return dense_dc(g.c[ci], dimg + rl.comp_off[ci], q.row, q.col);
}
template <class Sink>
__device__ __forceinline__ void emit_dc(int dcv, int last_dc, Sink &sink)
{
  int temp = dcv - last_dc, temp2 = temp;
  if (temp < 0) { temp = -temp; temp2--; }
  sink.dc(nbits_of(temp), temp2);
}
// encode_one_block (jchuff.c:563-661) / htest_one_block (:812-878) for scan block t from its record
template <class Sink>
__device__ __forceinline__ void walk_seq_rec(const Geom &g, const ScanDesc &sd, const uint8_t *__restrict__ sym, const int16_t *__restrict__ dcq, const RecLayout &rl,
                                             int img, long long t, Sink &sink)
{
  const ScanPos sp = scan_coords(g, sd, t);
  const int row = sp.row, col = sp.col;
  const int ci = sd.ci[sp.sci];
  const CompGeom &c = g.c[ci];
  const int16_t *dimg = dcq + (size_t)img * rl.per_image;
  const bool real = row < c.hib && col < c.wib;
  const size_t ridx = (size_t)img * rl.per_image + rl.comp_off[ci] + (real ? (size_t)row * c.wib + col : (size_t)0);
#if SYMREC_SPLIT
  const uint4 *r4 = reinterpret_cast<const uint4 *>(sym + ridx * (SYMREC_BYTES / 2));
  const uint4 *r4hi = reinterpret_cast<const uint4 *>(sym + (size_t)rl.sym_hi + ridx * (SYMREC_BYTES / 2)) - 4;      // words 16..31 = pieces 4..7
#else
  const uint4 *r4 = reinterpret_cast<const uint4 *>(sym + ridx * SYMREC_BYTES);
  const uint4 *r4hi = r4;
#endif
  uint4 q0 = make_uint4(1u, 0u, 0u, 0u);                       // a dummy block: one entry, EOB
  if (real) q0 = r4[0];
  emit_dc(dense_dc(c, dimg + rl.comp_off[ci], row, col), prev_dc_dense(g, sd, dimg, rl, sp), sink);
  if (q0.x & 0x80u) {
    // more symbols than a record holds: the coefficient block itself
    const int16_t *blk = c.coef + (((size_t)img * c.hpad + row) * c.wpad + col) * 64;
    int r = 0;
    for (int p = 1; p < 64; p++) {
      const int val = blk[p];
      if (val == 0) { r++; continue; }
      while (r > 15) { sink.ac(0xF0, 0, 0); r -= 16; }
      int temp = val, temp2 = val;
      if (temp < 0) { temp = -temp; temp2--; }
      const int nb = nbits_of(temp);
      sink.ac((r << 4) + nb, nb, temp2);
      r = 0;
    }
    if (r > 0) sink.ac(0, 0, 0);
    return;
  }
  const int n = (int)(q0.x & 0x7Fu);                          // entries at words 1..n, stream order = descending word index
#pragma unroll 1
  for (int v = n >> 2; v > 0; v--) {
    const uint4 q = v < 4 ? r4[v] : r4hi[v];
    const unsigned e[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int j = 3; j >= 0; j--) if (4 * v + j <= n) sink.ac((int)(e[j] & 0xFFu), (int)(e[j] & 15u), (int)(e[j] >> 16));
  }
  if (n >= 3) sink.ac((int)(q0.w & 0xFFu), (int)(q0.w & 15u), (int)(q0.w >> 16));
  if (n >= 2) sink.ac((int)(q0.z & 0xFFu), (int)(q0.z & 15u), (int)(q0.z >> 16));
  if (n >= 1) sink.ac((int)(q0.y & 0xFFu), (int)(q0.y & 15u), (int)(q0.y >> 16));
}

// ---------------------------------------------------------------------
// statistics pass (encode_mcu_gather, jchuff.c:886-915)
// ---------------------------------------------------------------------
// shared-memory histogram increment (warp-aggregating the atomics per counter was measured slower).  A few symbols
// (EOB, 0x01, 0x11, 0x02) make up most of a scan, so the lanes of a warp mostly hit the same few counters; keeping
// GATHER_COPIES copies of the histograms per CTA (a thread uses copy lane mod copies) is a build-time option; the
// per-scan kernels' copies are 8 KB each, so more copies cost occupancy there.  Default 1 (not re-measured on H100).
#ifndef GATHER_COPIES
#define GATHER_COPIES 1
#endif
#ifndef GATHER_COPIES_SCAN
#define GATHER_COPIES_SCAN 1
#endif
// blocks per CTA = GATHER_TILES * 256: zeroing and flushing the copies is paid once per CTA
#ifndef GATHER_TILES
#define GATHER_TILES 4
#endif
__device__ __forceinline__ void hist_inc(unsigned *addr)
{
  atomicAdd(addr, 1u);
}
struct HistSink {
  unsigned *dc_hist, *ac_hist; int bad; int maxbits;        // maxbits = data_precision + 2 (jchuff.c:819,836,865)
  __device__ void dc(int nb, int) { if (nb > maxbits + 1) bad = 1; hist_inc(&dc_hist[nb]); }
  __device__ void ac(int sym, int nb, int) { if (nb > maxbits) bad = 1; hist_inc(&ac_hist[sym]); }
};

// nz_rec: the side records holding every block's final non-zero positions (after the AC trellis), or nullptr: the walk
// then touches only those coefficients (and the 32-byte sectors they sit in) instead of the whole 128-byte block
__global__ void __launch_bounds__(256) k_gather_seq(Geom g, ScanDesc sd, const DcRec *__restrict__ nz_rec, const uint8_t *__restrict__ sym, const int16_t *__restrict__ dcq,
                                                    RecLayout rl, uint32_t *__restrict__ hist, uint32_t *__restrict__ status)
{
  __shared__ unsigned sh[GATHER_COPIES_SCAN][HIST_SLOTS * HIST_BINS];
  int img = blockIdx.y;
  for (int i = threadIdx.x; i < GATHER_COPIES_SCAN * HIST_SLOTS * HIST_BINS; i += blockDim.x) (&sh[0][0])[i] = 0;
  __syncthreads();
#pragma unroll 1
  for (int tile = 0; tile < GATHER_TILES; tile++) {
    long long t = ((long long)blockIdx.x * GATHER_TILES + tile) * blockDim.x + threadIdx.x;
    if (t >= sd.nblocks) break;
    unsigned *mine = sh[threadIdx.x % GATHER_COPIES_SCAN];
    if (sym) {                                         // symbol records (a scan script with several sequential scans: per-scan counts)
      const CompGeom &c = g.c[sd.ci[sd.k_comp[(int)(t % sd.bim)]]];
      HistSink sink{mine + c.dc_tbl * HIST_BINS, mine + (4 + c.ac_tbl) * HIST_BINS, 0, g.max_coef_bits};
      walk_seq_rec(g, sd, sym, dcq, rl, img, t, sink);
      if (sink.bad) atomicOr(&status[img], 2u);
      continue;
    }
    int sci, k; long long mcu;
    const int16_t *blk = block_ptr(g, sd, img, t, sci, mcu, k);
    int last = prev_dc(g, sd, img, t, sci, mcu, k);
    const CompGeom &c = g.c[sd.ci[sci]];
    HistSink sink{mine + c.dc_tbl * HIST_BINS, mine + (4 + c.ac_tbl) * HIST_BINS, 0, g.max_coef_bits};
    if (SEQ_SPARSE_STATS && nz_rec) walk_seq_sparse(blk, block_nzmask(g, sd, nz_rec, rl, img, sci, mcu, k), last, sink);
    else walk_seq_block(blk, last, sink);
    if (sink.bad) atomicOr(&status[img], 2u);          // JERR_BAD_DCT_COEF
  }
  __syncthreads();
  uint32_t *gh = hist + (size_t)img * HIST_SLOTS * HIST_BINS;
  for (int i = threadIdx.x; i < HIST_SLOTS * HIST_BINS; i += blockDim.x) {
    unsigned v = 0;
#pragma unroll
    for (int cp = 0; cp < GATHER_COPIES_SCAN; cp++) v += sh[cp][i];
    if (v) atomicAdd(&gh[i], v);
  }
}
// Trellis-phase statistics: every component as its own non-interleaved scan
// (jcmaster.c:443-467), all components of all images in one launch;
// histogram set index = img*nc + ci.
// GATHER_STAGE: the CTA's 256 blocks arrive through shared memory -- 16-byte pieces in the order they lie in memory (8
// consecutive lanes fetch one block's 128 bytes: 4 lines per request instead of 32), stored with the piece index XORed
// by the block's low bits so that the per-thread read-back of whole blocks is conflict-free.
#ifndef GATHER_STAGE
#define GATHER_STAGE 0
#endif
__global__ void __launch_bounds__(256) k_gather_comp(Geom g, RestartSpec rs, uint32_t *__restrict__ hist, uint32_t *__restrict__ status)
{
  __shared__ unsigned sh[GATHER_COPIES][2 * HIST_BINS];
  __shared__ __align__(16) uint4 stg[GATHER_STAGE ? 256 * 8 : 1];
  const int ci = blockIdx.y % g.nc, img = blockIdx.y / g.nc;
  const CompGeom &c = g.c[ci];
  long long nblk = (long long)c.wib * c.hib;
  if ((long long)blockIdx.x * GATHER_TILES * blockDim.x >= nblk) return;
  for (int i = threadIdx.x; i < GATHER_COPIES * 2 * HIST_BINS; i += blockDim.x) (&sh[0][0])[i] = 0;
  __syncthreads();
  const int16_t *base = c.coef + (size_t)img * c.blocks_per_image * 64;
#pragma unroll 1
  for (int tile = 0; tile < GATHER_TILES; tile++) {
    const long long t0 = ((long long)blockIdx.x * GATHER_TILES + tile) * blockDim.x;
    if (t0 >= nblk) break;
    if (GATHER_STAGE) {
      if (tile) __syncthreads();                             // the previous tile's blocks have been read
#pragma unroll
      for (int i = 0; i < 8; i++) {
        const int q = i * 256 + threadIdx.x, bq = q >> 3, part = q & 7;
        const long long tb = t0 + bq;
        if (tb < nblk) {
          const int rowb = (int)(tb / c.wib), colb = (int)(tb - (long long)rowb * c.wib);
          stg[bq * 8 + (part ^ (bq & 7))] = reinterpret_cast<const uint4 *>(base + ((size_t)rowb * c.wpad + colb) * 64)[part];
        }
      }
      __syncthreads();
    }
    const long long t = t0 + threadIdx.x;
    if (t < nblk) {
      int row = (int)(t / c.wib), col = (int)(t - (long long)row * c.wib);
      const int16_t *blk = base + ((size_t)row * c.wpad + col) * 64;
      int last = 0;
      const long long ri = rs.in_rows > 0 ? min((long long)rs.in_rows * c.wib, 65535LL) : rs.interval;      // per_scan_setup, jcmaster.c:594-599
      if (t > 0 && !(ri && t % ri == 0)) { int pr = col > 0 ? row : row - 1, pc = col > 0 ? col - 1 : c.wib - 1; last = base[((size_t)pr * c.wpad + pc) * 64]; }
      unsigned *mine = sh[threadIdx.x % GATHER_COPIES];
      HistSink sink{mine, mine + HIST_BINS, 0, g.max_coef_bits};
      if (GATHER_STAGE) { const uint4 *mb = stg + threadIdx.x * 8; const int sw = threadIdx.x & 7; walk_seq_chunks([&](int v) { return mb[v ^ sw]; }, last, sink); }
      else walk_seq_block(blk, last, sink);
      if (sink.bad) atomicOr(&status[img], 2u);
    }
  }
  __syncthreads();
  uint32_t *gh = hist + ((size_t)img * g.nc + ci) * HIST_SLOTS * HIST_BINS;
  for (int i = threadIdx.x; i < HIST_BINS; i += blockDim.x) {
    unsigned d = 0, a = 0;
#pragma unroll
    for (int cp = 0; cp < GATHER_COPIES; cp++) { d += sh[cp][i]; a += sh[cp][HIST_BINS + i]; }
    if (d) atomicAdd(&gh[c.dc_tbl * HIST_BINS + i], d);
    if (a) atomicAdd(&gh[(4 + c.ac_tbl) * HIST_BINS + i], a);
  }
}
void launch_gather_comp(const Geom &g, const RestartSpec &rs, uint32_t *hist, uint32_t *status, int n, cudaStream_t s)
{
  long long mb = 0;
  for (int ci = 0; ci < g.nc; ci++) mb = max(mb, (long long)g.c[ci].wib * g.c[ci].hib);
  dim3 grid((unsigned)((mb + 256 * GATHER_TILES - 1) / (256 * GATHER_TILES)), n * g.nc);
  k_gather_comp<<<grid, 256, 0, s>>>(g, rs, hist, status);
  LAUNCHED();
}

// k_gather_comp's DC half from the dense plain-quantized DC values the tiled forward kernel left (it counted the AC
// half): the same scan order, restart rule and JERR_BAD_DCT_COEF check, 2 bytes read per block
__global__ void __launch_bounds__(256) k_gather_comp_dc(Geom g, RestartSpec rs, const int16_t *__restrict__ dcq, RecLayout rl, uint32_t *__restrict__ hist, uint32_t *__restrict__ status)
{
  __shared__ unsigned sdc[4][17];                              // |DC difference| < 2^16: sizes 0..16
  const int ci = blockIdx.y % g.nc, img = blockIdx.y / g.nc;
  const CompGeom &c = g.c[ci];
  const long long nblk = (long long)c.wib * c.hib;
  if ((long long)blockIdx.x * GATHER_TILES * blockDim.x >= nblk) return;
  for (int i = threadIdx.x; i < 4 * 17; i += blockDim.x) (&sdc[0][0])[i] = 0;
  __syncthreads();
  const int16_t *d = dcq + (size_t)img * rl.per_image + rl.comp_off[ci];
  const long long ri = rs.in_rows > 0 ? min((long long)rs.in_rows * c.wib, 65535LL) : rs.interval;      // per_scan_setup, jcmaster.c:594-599
  bool bad = false;
#pragma unroll 1
  for (int tile = 0; tile < GATHER_TILES; tile++) {
    const long long t = ((long long)blockIdx.x * GATHER_TILES + tile) * blockDim.x + threadIdx.x;
    if (t >= nblk) break;
    const int last = (t > 0 && !(ri && t % ri == 0)) ? d[t - 1] : 0;
    const int nb = nbits_of(abs((int)d[t] - last));
    bad |= nb > g.max_coef_bits + 1;
    atomicAdd(&sdc[threadIdx.x & 3][nb], 1u);
  }
  if (bad) atomicOr(&status[img], 2u);                        // JERR_BAD_DCT_COEF (jchuff.c:836)
  __syncthreads();
  if (threadIdx.x < 17) {
    const unsigned v = sdc[0][threadIdx.x] + sdc[1][threadIdx.x] + sdc[2][threadIdx.x] + sdc[3][threadIdx.x];
    if (v) atomicAdd(&hist[(((size_t)img * g.nc + ci) * HIST_SLOTS + c.dc_tbl) * HIST_BINS + threadIdx.x], v);
  }
}
void launch_gather_comp_dc(const Geom &g, const RestartSpec &rs, const int16_t *dcq, const RecLayout &rl, uint32_t *hist, uint32_t *status, int n, cudaStream_t s)
{
  long long mb = 0;
  for (int ci = 0; ci < g.nc; ci++) mb = max(mb, (long long)g.c[ci].wib * g.c[ci].hib);
  dim3 grid((unsigned)((mb + 256 * GATHER_TILES - 1) / (256 * GATHER_TILES)), n * g.nc);
  k_gather_comp_dc<<<grid, 256, 0, s>>>(g, rs, dcq, rl, hist, status);
  LAUNCHED();
}

void launch_gather_seq(const Geom &g, const ScanDesc &sd, const DcRec *nz_rec, const uint8_t *sym, const int16_t *dcq, const RecLayout &rl, uint32_t *hist, uint32_t *status, int n, cudaStream_t s)
{
  dim3 grid((unsigned)((sd.nblocks + 256 * GATHER_TILES - 1) / (256 * GATHER_TILES)), n);
  k_gather_seq<<<grid, 256, 0, s>>>(g, sd, nz_rec, sym, dcq, rl, hist, status);
  LAUNCHED();
}

// The DC half of a sequential scan's statistics, from the dense DC values (the AC half was counted by the AC trellis
// back-track); dummy blocks add their EOB here.  GATHER_TILES * 256 scan blocks per CTA.
__global__ void __launch_bounds__(256) k_gather_seq_dc(Geom g, ScanDesc sd, const int16_t *__restrict__ dcq, RecLayout rl, uint32_t *__restrict__ hist, uint32_t *__restrict__ status)
{
  __shared__ unsigned sdc[4][4][20], seob[4];
  const int img = blockIdx.y;
  for (int i = threadIdx.x; i < 4 * 4 * 20; i += blockDim.x) (&sdc[0][0][0])[i] = 0;
  if (threadIdx.x < 4) seob[threadIdx.x] = 0;
  __syncthreads();
  const int16_t *dimg = dcq + (size_t)img * rl.per_image;
#pragma unroll 1
  for (int tile = 0; tile < GATHER_TILES; tile++) {
    const long long t = ((long long)blockIdx.x * GATHER_TILES + tile) * blockDim.x + threadIdx.x;
    if (t >= sd.nblocks) break;
    const ScanPos sp = scan_coords(g, sd, t);
    const int row = sp.row, col = sp.col;
    const int ci = sd.ci[sp.sci];
    const CompGeom &c = g.c[ci];
    int temp = dense_dc(c, dimg + rl.comp_off[ci], row, col) - prev_dc_dense(g, sd, dimg, rl, sp);
    if (temp < 0) temp = -temp;
    const int nb = nbits_of(temp);
    if (nb > g.max_coef_bits + 1) atomicOr(&status[img], 2u);          // JERR_BAD_DCT_COEF (jchuff.c:836)
    atomicAdd(&sdc[threadIdx.x & 3][c.dc_tbl][min(nb, 19)], 1u);
    if (!(row < c.hib && col < c.wib)) atomicAdd(&seob[c.ac_tbl], 1u);
  }
  __syncthreads();
  uint32_t *gh = hist + (size_t)img * HIST_SLOTS * HIST_BINS;
  if (threadIdx.x < 80) {
    const int slot = threadIdx.x / 20, b = threadIdx.x % 20;
    const unsigned v = sdc[0][slot][b] + sdc[1][slot][b] + sdc[2][slot][b] + sdc[3][slot][b];
    if (v) atomicAdd(&gh[slot * HIST_BINS + b], v);
  } else if (threadIdx.x < 84) {
    const int slot = threadIdx.x - 80;
    if (seob[slot]) atomicAdd(&gh[(4 + slot) * HIST_BINS], seob[slot]);
  }
}
void launch_gather_seq_dc(const Geom &g, const ScanDesc &sd, const int16_t *dcq, const RecLayout &rl, uint32_t *hist, uint32_t *status, int n, cudaStream_t s)
{
  dim3 grid((unsigned)((sd.nblocks + 256 * GATHER_TILES - 1) / (256 * GATHER_TILES)), n);
  k_gather_seq_dc<<<grid, 256, 0, s>>>(g, sd, dcq, rl, hist, status); LAUNCHED();
}

// =====================================================================
// optimal Huffman table from counts: jpeg_gen_optimal_table (jchuff.c:947-1106)
// + jpeg_make_c_derived_tbl (jchuff.c:231-318).  One warp per (image, slot).
// The two-smallest search of :997-1011 ("<=" => the LARGER index wins ties,
// c1 = overall minimum, c2 = minimum of the rest) runs across the warp; the
// code-size chains (:1021-1034) are replaced by a reverse sweep over the
// recorded merge list, which yields the same leaf depths.
// =====================================================================
// blockIdx.y enumerates histogram/table SETS (one per image, or one per
// (image, component) in the trellis phase); masks.m[set % masks.period] says which of
// the 8 slots of that set are to be built.
__global__ void __launch_bounds__(32) k_gen_tables(const uint32_t *__restrict__ hist, DevHuff *__restrict__ tabs,
                                                   size_t tabs_set_stride, SlotMasks masks)
{
  int img = blockIdx.y, slot = blockIdx.x, lane = threadIdx.x;
  if (!((masks.m[img % masks.period] >> slot) & 1)) return;
  __shared__ long long freq[257];
  __shared__ short nz_index[257];
  __shared__ short m1[257], m2[257];
  __shared__ int depth[257];
  __shared__ int nnz_s;
  const uint32_t *h = hist + ((size_t)img * HIST_SLOTS + slot) * HIST_BINS;
  if (lane == 0) {
    int n = 0;
    for (int i = 0; i < 257; i++) {
      long long f = (i == 256) ? 1 : (long long)(h[i]);
      if (f) { nz_index[n] = (short)i; freq[n] = f; n++; }
    }
    nnz_s = n;
  }
  __syncwarp();
  const int nnz = nnz_s;
  int nmerge = 0;
  for (;;) {
    // key = (freq << 9) | (511 - idx): min key == smallest freq, largest index on ties
    unsigned long long best = ~0ull;
    for (int i = lane; i < nnz; i += 32) {
      long long f = freq[i];
      if (f <= 1000000000LL) { unsigned long long key = ((unsigned long long)f << 9) | (unsigned)(511 - i); if (key < best) best = key; }
    }
    for (int o = 16; o; o >>= 1) { unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o); if (other < best) best = other; }
    if (best == ~0ull) break;
    int c1 = 511 - (int)(best & 511);
    unsigned long long best2 = ~0ull;
    for (int i = lane; i < nnz; i += 32) {
      long long f = freq[i];
      if (i != c1 && f <= 1000000000LL) { unsigned long long key = ((unsigned long long)f << 9) | (unsigned)(511 - i); if (key < best2) best2 = key; }
    }
    for (int o = 16; o; o >>= 1) { unsigned long long other = __shfl_xor_sync(0xffffffffu, best2, o); if (other < best2) best2 = other; }
    if (best2 == ~0ull) break;
    int c2 = 511 - (int)(best2 & 511);
    if (lane == 0) { freq[c1] += freq[c2]; freq[c2] = 1000000001LL; m1[nmerge] = (short)c1; m2[nmerge] = (short)c2; }
    nmerge++;
    __syncwarp();
  }
  if (lane == 0) {
    DevHuff *out = reinterpret_cast<DevHuff *>(reinterpret_cast<char *>(tabs) + (size_t)img * tabs_set_stride) + slot;
    for (int i = 0; i < nnz; i++) depth[i] = 0;
    for (int t = nmerge - 1; t >= 0; t--) { int d = depth[m1[t]] + 1; depth[m1[t]] = d; depth[m2[t]] = d; }
    unsigned char bits[33]; int bit_pos[33];
    for (int i = 0; i <= 32; i++) bits[i] = 0;
    for (int i = 0; i < nnz; i++) { int d = depth[i] > 32 ? 32 : depth[i]; bits[d]++; }
    int p = 0;
    for (int i = 1; i <= 32; i++) { bit_pos[i] = p; p += bits[i]; }
    int i;
    for (i = 32; i > 16; i--) {
      while (bits[i] > 0) {
        int j = i - 2;
        while (bits[j] == 0) j--;
        bits[i] -= 2; bits[i - 1]++; bits[j + 1] += 2; bits[j]--;
      }
    }
    while (bits[i] == 0) i--;
    bits[i]--;
    for (int l = 0; l <= 16; l++) out->bits[l] = bits[l];
    for (int s = 0; s < nnz - 1; s++) { int d = depth[s] > 32 ? 32 : depth[s]; out->huffval[bit_pos[d]] = (uint8_t)nz_index[s]; bit_pos[d]++; }
    // derived table (C.1-C.3)
    for (int s = 0; s < 256; s++) { out->code[s] = 0; out->size[s] = 0; }
    int nsym = 0; unsigned code = 0;
    for (int l = 1; l <= 16; l++) {
      for (int c = 0; c < bits[l]; c++) { int sym = out->huffval[nsym++]; out->code[sym] = (uint16_t)code; out->size[sym] = (uint8_t)l; code++; }
      code <<= 1;
    }
    out->nsym16 = (uint16_t)nsym; out->nsym = (uint8_t)nsym;
  }
}
void launch_gen_tables(const uint32_t *hist, DevHuff *tabs, size_t tabs_set_stride, const SlotMasks &masks, int nsets, cudaStream_t s)
{
  dim3 grid(HIST_SLOTS, nsets);
  k_gen_tables<<<grid, 32, 0, s>>>(hist, tabs, tabs_set_stride, masks);
  LAUNCHED();
}

// jcphuff.c:257-264: in trellis passes every symbol 16*i+j (i<16, j<12) starts with count 1
__global__ void k_seed_hist(uint32_t *hist, int slot)
{
  int img = blockIdx.x, t = threadIdx.x;
  if ((t & 15) < 12) hist[((size_t)img * HIST_SLOTS + slot) * HIST_BINS + t] = 1;
}
void launch_seed_hist(uint32_t *hist, int slot, int n, cudaStream_t s) { k_seed_hist<<<n, 256, 0, s>>>(hist, slot); LAUNCHED(); }

// =====================================================================
// trellis quantization, AC part: quantize_trellis (jcdctmgr.c:936-1330).
//   phase 1: lambda from the block's norm, accumulated zero distortion (zigzag order, serial fp32), an entry for
//            every position whose plain-quantized value is non-zero;
//   phase 2: for each entry the best (predecessor, candidate) pair, strict '<' in (predecessor, candidate) order
//            (:1157-1184);
//   phase 3: best end-of-block position (:1187-1207) and back-tracking (:1211-1222).
// The default option set runs on k_trellis_ac3 (below, with the sorting kernels); the optional modes (two AC bands,
// repeated rounds, EOB-run optimisation, table re-fitting) on the literal band kernel that follows.
// =====================================================================
// ---------------------------------------------------------------------
// Optional trellis mode use_scans_in_trellis (jcmaster.c:451-467): the AC coefficients of a component are requantized
// in two passes, zigzag positions 1..trellis_freq_split and the rest, each with Huffman tables gathered just before
// it.  quantize_trellis then works on the band [Ss, Se] only (jcdctmgr.c:975-980, :1121-1222): zero distortion and
// runs start at position Ss-1, the end-of-block choice is made at Se, and coefficients outside the band are left
// alone.  One thread per block, the reference's (predecessor, candidate) loop order kept literally; an API-only
// option, so this kernel is written for exactness, not speed.  Also (re)writes lambda_dc for the DC trellis that
// follows each pass, from the natural-order norm recomputed here (:1026-1035).
// ---------------------------------------------------------------------
// qimg: per-image quantization tables [img][4][64] (natural order) that trellis_q_opt has re-fitted, or nullptr for the
// batch's tables; eo: per real block {zero-distortion cost of blanking the band, best cost without the EOB symbol,
// has_eob} for the block-level EOB-run pass of trellis_eob_opt (k_trellis_eob_rows), or nullptr.
__global__ void __launch_bounds__(128) k_trellis_ac_band(Geom g, const TrellisConsts *__restrict__ tc,
                                                         const DevHuff *__restrict__ tabs, size_t tabs_set_stride,
                                                         DcRec *__restrict__ rec, RecLayout rl, int Ss, int Se,
                                                         const uint16_t *__restrict__ qimg, float4 *__restrict__ eo)
{
  const int ci = blockIdx.y % g.nc, img = blockIdx.y / g.nc;
  const CompGeom &c = g.c[ci];
  __shared__ float swz[64];
  __shared__ int sq8[64];
  __shared__ uint8_t acsi[256];
  const long long nblk = (long long)c.wib * c.hib;
  if ((long long)blockIdx.x * blockDim.x >= nblk) return;
  tc = qset_of(tc, g, img);
  {
    const DevHuff *ac = reinterpret_cast<const DevHuff *>(reinterpret_cast<const char *>(tabs) + (size_t)blockIdx.y * tabs_set_stride) + (4 + c.ac_tbl);
    for (int i = threadIdx.x; i < 256; i += blockDim.x) acsi[i] = ac->size[i];
    if (threadIdx.x < 64) {
      if (qimg) {                                                // jcdctmgr.c:1017-1021 on this image's current table
        const int Q = qimg[((size_t)img * 4 + c.qt) * 64 + c_zz[threadIdx.x]];
        swz[threadIdx.x] = (float)(1.0 / (double)(Q * Q)); sq8[threadIdx.x] = 8 * Q;
      } else { swz[threadIdx.x] = tc->w_zz[c.qt][threadIdx.x]; sq8[threadIdx.x] = tc->q8_zz[c.qt][threadIdx.x]; }
    }
  }
  __syncthreads();
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nblk) return;
  const int by = (int)(t / c.wib), bx = (int)(t - (long long)by * c.wib);
  const size_t blk = ((size_t)img * c.hpad + by) * c.wpad + bx;
  const int16_t *raw16 = c.raw + blk * 64;
  int16_t *o16 = c.coef + blk * 64;
  const size_t ridx = (size_t)img * rl.per_image + rl.comp_off[ci] + (size_t)t;
  float lambda;
  {
    float nsum = 0.0f;
    for (int nat = 1; nat < 64; nat++) { const int v = raw16[c_izz[nat]]; nsum += (float)(v * v); }
    const float norm = (float)((double)nsum / 63.0);
    if (tc->use_norm) lambda = (float)(tc->p1 / (tc->p2 + (double)norm));
    else lambda = tc->lambda_const;
    rec[ridx].lambda_dc = lambda * swz[0];
  }
  const int maxq = (1 << tc->max_coef_bits) - 1;
  float azd[64], acc[64];
  int16_t cur[64];
  uint8_t rs[64];
  for (int i = Ss; i <= Se; i++) cur[i] = o16[i];
  azd[Ss - 1] = 0.0f; acc[Ss - 1] = 0.0f; cur[Ss - 1] = 0; rs[Ss - 1] = 0;
  const int zrl = acsi[0xF0];
  for (int i = Ss; i <= Se; i++) {
    const int rawv = raw16[i], sign = rawv >> 31, x = abs(rawv), q = sq8[i];
    azd[i] = (float)(x * x) * lambda * swz[i] + azd[i - 1];
    rs[i] = 0;
    int qval = (x + q / 2) / q;
    if (qval == 0) { cur[i] = 0; acc[i] = 1e38f; continue; }
    if (qval > maxq) qval = maxq;
    const int nc = nbits_of(qval);
    acc[i] = 1e38f;
    for (int j = Ss - 1; j < i; j++) {
      if (j != Ss - 1 && cur[j] == 0) continue;
      int zero_run = i - 1 - j;
      if ((zero_run >> 4) && zrl == 0) continue;
      const int run_bits = (zero_run >> 4) * zrl;
      zero_run &= 15;
      for (int k = 0; k < nc; k++) {
        const int cand = (k < nc - 1) ? (2 << k) - 1 : qval;
        const int coef_bits = acsi[16 * zero_run + k + 1];
        if (coef_bits == 0) continue;
        const int delta = cand * q - x;
        const float dist = (float)(delta * delta) * lambda * swz[i];
        float cost = (float)(coef_bits + (k + 1) + run_bits) + dist;
        cost += (azd[i - 1] - azd[j]) + acc[j];
        if (cost < acc[i]) { cur[i] = (int16_t)((cand ^ sign) - sign); acc[i] = cost; rs[i] = (uint8_t)j; }
      }
    }
  }
  int last = Ss - 1;
  float best = azd[Se] + (float)acsi[0];
  float best_skip = azd[Se];                                   // :1189-1190 cost_all_zeros, best_cost_skip
  for (int i = Ss; i <= Se; i++) {
    if (cur[i] != 0) {
      float cst = acc[i] + azd[Se] - azd[i];
      const float wo_eob = cst;
      if (i < Se) cst += (float)acsi[0];
      if (cst < best) { best = cst; last = i; best_skip = wo_eob; }
    }
  }
  if (eo) eo[ridx] = make_float4(azd[Se], best_skip, __int_as_float((last < Se) + (last == Ss - 1)), 0.f);   // :1209 has_eob
  for (int i = Se; i >= Ss; ) {
    while (i > last) { cur[i] = 0; i--; }
    if (i < Ss) break;
    last = rs[i];
    i--;
  }
  unsigned long long bits = 0;
  for (int i = Ss; i <= Se; i++) { o16[i] = cur[i]; if (cur[i]) bits |= 1ull << i; }
  const unsigned long long bandmask = ((Se >= 63 ? ~0ull : ((1ull << (Se + 1)) - 1ull))) & ~((1ull << Ss) - 1ull);
  rec[ridx].nzmask = (rec[ridx].nzmask & ~bandmask) | bits;
}
void launch_trellis_ac_band(const Geom &g, const TrellisConsts *tc, const DevHuff *tabs, size_t tabs_set_stride,
                            DcRec *rec, const RecLayout &rl, int Ss, int Se, const uint16_t *qimg, float4 *eo, int n, cudaStream_t s)
{
  long long mb = 0;
  for (int ci = 0; ci < g.nc; ci++) mb = max(mb, (long long)g.c[ci].wib * g.c[ci].hib);
  dim3 grid((unsigned)((mb + 127) / 128), n * g.nc);
  k_trellis_ac_band<<<grid, 128, 0, s>>>(g, tc, tabs, tabs_set_stride, rec, rl, Ss, Se, qimg, eo);
  LAUNCHED();
}

// ---------------------------------------------------------------------
// trellis_eob_opt (jcdctmgr.c:981-996, :1224-1297): after the per-block search, a second dynamic program along each
// block row decides which blocks to blank so that runs of all-zero blocks can share one EOBRUN symbol.  One warp per
// (image, component, block row); the predecessor loop of :1232-1254 runs across the lanes (each lane keeps the first
// minimum of its own ascending stripe, the warp then takes the smallest cost with ties to the smaller index, which is
// the reference's strict-'<' scan order); the four per-block arrays live in the scratch `es` (16 bytes per block).
// ---------------------------------------------------------------------
// slot b of a row's scratch: accumulated_zero_block_cost[b+1], accumulated_block_cost[b+1], requires_eob[b+1] and
// block_run_start[b]; index 0 of the three arrays is the constant initial state {0, 0, 0} (:991-995)
struct EobState { float zero, cost; int start, req; };
__global__ void __launch_bounds__(32) k_trellis_eob_rows(Geom g, const DevHuff *__restrict__ tabs, size_t tabs_set_stride,
                                                        DcRec *__restrict__ rec, RecLayout rl, int Ss, int Se,
                                                        const float4 *__restrict__ eo, EobState *__restrict__ es /* one slot per real block */)
{
  const int ci = blockIdx.y % g.nc, img = blockIdx.y / g.nc;
  const CompGeom &c = g.c[ci];
  const int row = blockIdx.x;
  if (row >= c.hib) return;
  const int n = c.wib, lane = threadIdx.x;
  __shared__ uint8_t acsi[256];
  {
    const DevHuff *ac = reinterpret_cast<const DevHuff *>(reinterpret_cast<const char *>(tabs) + (size_t)blockIdx.y * tabs_set_stride) + (4 + c.ac_tbl);
    for (int i = lane; i < 256; i += 32) acsi[i] = ac->size[i];
  }
  __syncwarp();
  const size_t rbase = (size_t)img * rl.per_image + rl.comp_off[ci] + (size_t)row * n;
  const float4 *e = eo + rbase;
  EobState *st = es + rbase;
  auto state = [&](int i, float &zero, float &cost, int &req) {
    if (i == 0) { zero = 0.f; cost = 0.f; req = 0; }
    else { const EobState p = st[i - 1]; zero = p.zero; cost = p.cost; req = p.req; }
  };
  // the smallest cost over the lanes, ties to the smaller predecessor index (= the first minimum of the ascending scan)
  auto warp_first_min = [&](float &best, int &best_i) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, off); const int oi = __shfl_xor_sync(0xffffffffu, best_i, off);
      if (oi >= 0 && (best_i < 0 || ob < best || (ob == best && oi < best_i))) { best = ob; best_i = oi; }
    }
  };
  float zb = 0.f;                                              // accumulated_zero_block_cost[bi]
  for (int bi = 0; bi < n; bi++) {
    const float4 me = e[bi];
    const int has_eob = __float_as_int(me.z);
    float best = 1e38f; int best_i = -1;
    if (has_eob != 2) {                                        // :1232-1254
      for (int i = lane; i <= bi; i += 32) {
        float pz, pc; int pr; state(i, pz, pc, pr);
        if (pr == 2) continue;
        float cst = me.y;                                       // cost of coding a non-zero block
        cst += zb; cst -= pz; cst += pc;
        const int run = bi - i + pr, nb = nbits_of(run);
        cst += (float)(acsi[16 * nb] + nb);
        if (cst < best) { best = cst; best_i = i; }
      }
      warp_first_min(best, best_i);
    }
    __syncwarp();
    const float znext = zb + me.x;
    if (lane == 0) {
      EobState nx; nx.zero = znext; nx.req = has_eob; nx.cost = best_i >= 0 ? best : 0.f; nx.start = best_i >= 0 ? best_i : 0;
      st[bi] = nx;
    }
    zb = znext;
    __syncwarp();
  }
  // :1258-1276 where the last run of blank blocks starts
  int last_block = n;
  {
    float best = 1e38f; int best_i = -1;
    for (int i = lane; i <= n; i += 32) {
      float pz, pc; int pr; state(i, pz, pc, pr);
      if (pr == 2) continue;
      float cst = 0.0f;
      cst += zb; cst -= pz;
      const int run = n - i + pr, nb = nbits_of(run);
      cst += (float)(acsi[16 * nb] + nb);
      if (cst < best) { best = cst; best_i = i; }
    }
    warp_first_min(best, best_i);
    if (best_i >= 0) last_block = best_i;
  }
  // :1277-1292 back-track; blanked blocks lose the band's coefficients (the lanes clear one block together)
  last_block--;
  int bi = n - 1;
  const unsigned long long bandmask = ((Se >= 63 ? ~0ull : ((1ull << (Se + 1)) - 1ull))) & ~((1ull << Ss) - 1ull);
  while (bi >= 0) {
    while (bi > last_block) {
      int16_t *blk = c.coef + (((size_t)img * c.hpad + row) * c.wpad + bi) * 64;
      for (int k = Ss + lane; k <= Se; k += 32) blk[k] = 0;
      if (lane == 0) rec[rbase + bi].nzmask &= ~bandmask;
      bi--;
    }
    if (bi < 0) break;
    last_block = st[bi].start - 1;
    bi--;
  }
}
void launch_trellis_eob_rows(const Geom &g, const DevHuff *tabs, size_t tabs_set_stride, DcRec *rec, const RecLayout &rl, int Ss, int Se,
                             const float4 *eo, void *scratch, int n, cudaStream_t s)
{
  int mh = 0; for (int ci = 0; ci < g.nc; ci++) mh = max(mh, g.c[ci].hib);
  k_trellis_eob_rows<<<dim3(mh, n * g.nc), 32, 0, s>>>(g, tabs, tabs_set_stride, rec, rl, Ss, Se, eo, static_cast<EobState *>(scratch));
  LAUNCHED();
}

// ---------------------------------------------------------------------
// trellis_q_opt (jcdctmgr.c:1299-1306, jcmaster.c:1014-1030): per quantization table and coefficient position the
// sums of raw * kept and 8 * kept^2 over the blocks requantized since the last table update (64-bit integers: the
// reference adds the same integers in doubles, exactly), then the table entry becomes their rounded quotient.
// ---------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_qopt_sums(Geom g, long long *__restrict__ qsum /* [img][4][2][64] natural order */)
{
  __shared__ long long sh[2][64];
  const int ci = blockIdx.y % g.nc, img = blockIdx.y / g.nc;
  const CompGeom &c = g.c[ci];
  const long long nblk = (long long)c.wib * c.hib;
  if ((long long)blockIdx.x * blockDim.x >= nblk) return;
  if (threadIdx.x < 128) reinterpret_cast<long long *>(sh)[threadIdx.x] = 0;
  __syncthreads();
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < nblk) {
    const int by = (int)(t / c.wib), bx = (int)(t - (long long)by * c.wib);
    const size_t blk = ((size_t)img * c.hpad + by) * c.wpad + bx;
    const int16_t *raw16 = c.raw + blk * 64, *co = c.coef + blk * 64;
    for (int k = 1; k < 64; k++) {
      const int v = co[k];
      if (v) {
        atomicAdd(reinterpret_cast<unsigned long long *>(&sh[0][k]), (unsigned long long)(long long)((int)raw16[k] * v));
        atomicAdd(reinterpret_cast<unsigned long long *>(&sh[1][k]), (unsigned long long)(long long)(8 * v * v));
      }
    }
  }
  __syncthreads();
  if (threadIdx.x < 128) {
    const int which = threadIdx.x >> 6, k = threadIdx.x & 63;
    const long long v = sh[which][k];
    if (v) atomicAdd(reinterpret_cast<unsigned long long *>(&qsum[(((size_t)img * 4 + c.qt) * 2 + which) * 64 + c_zz[k]]), (unsigned long long)v);
  }
}
__global__ void k_qopt_update(long long *__restrict__ qsum, uint16_t *__restrict__ qimg, int n)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;          // (img, table, position)
  if (i >= n * 256) return;
  const int j = i & 63, it = i >> 6;
  if (j == 0) return;
  const long long ns = qsum[((size_t)it * 2 + 0) * 64 + j], nc2 = qsum[((size_t)it * 2 + 1) * 64 + j];
  if (nc2 != 0) {
    int q = (int)((double)ns / (double)nc2 + 0.5);
    if (q > 254) q = 254;
    if (q < 1) q = 1;
    qimg[(size_t)it * 64 + j] = (uint16_t)q;
  }
}
void launch_qopt_sums(const Geom &g, long long *qsum, int n, cudaStream_t s)
{
  long long mb = 0;
  for (int ci = 0; ci < g.nc; ci++) mb = max(mb, (long long)g.c[ci].wib * g.c[ci].hib);
  k_qopt_sums<<<dim3((unsigned)((mb + 127) / 128), n * g.nc), 128, 0, s>>>(g, qsum);
  LAUNCHED();
}
void launch_qopt_update(long long *qsum, uint16_t *qimg, int n, cudaStream_t s)
{
  k_qopt_update<<<(n * 256 + 255) / 256, 256, 0, s>>>(qsum, qimg, n);
  LAUNCHED();
}

// sorted side record of the AC trellis: {norm, block index inside the component, non-zero mask}
struct SRec { float norm; uint32_t lin; unsigned long long nzmask; };
static_assert(sizeof(SRec) == 16, "SRec layout");

// Counting sort of every (image, component)'s side records by their number of non-zero plain-quantized AC values,
// in decreasing order, so that the 32 blocks a warp of the trellis kernel works on have similar trip counts; four class
// boundaries per (image, component): [0, s0) more than 32 non-zeros, [s0, s1) mid_max+1..32, [s1, s2) 9..mid_max,
// [s2, nblk) at most 8.  Spread over several CTAs per (image, component) (one CTA each left most SMs idle behind the
// luma planes): k_sort_count adds each slice's counts per non-zero count to global counters, k_sort_scatter turns them
// into class offsets, reserves a range per count and slice with one global atomic each and writes the records.  The
// order inside a count is arbitrary (it only decides which blocks share a warp).  gcnt / gcur: [n*nc][64], zeroed.
#define SORT_SLICE 4096
__global__ void __launch_bounds__(256) k_sort_count(Geom g, const DcRec *__restrict__ rec, RecLayout rl, unsigned *__restrict__ gcnt)
{
  __shared__ unsigned cnt[64];
  const int ci = blockIdx.y % g.nc, img = blockIdx.y / g.nc;
  const CompGeom &c = g.c[ci];
  const long long nblk = (long long)c.wib * c.hib, b0 = (long long)blockIdx.x * SORT_SLICE;
  if (b0 >= nblk) return;
  const DcRec *r = rec + (size_t)img * rl.per_image + rl.comp_off[ci];
  if (threadIdx.x < 64) cnt[threadIdx.x] = 0;
  __syncthreads();
  const long long b1 = min(nblk, b0 + SORT_SLICE);
  for (long long b = b0 + threadIdx.x; b < b1; b += blockDim.x) atomicAdd(&cnt[63 - min((int)r[b].nz, 63)], 1u);
  __syncthreads();
  if (threadIdx.x < 64 && cnt[threadIdx.x]) atomicAdd(&gcnt[(size_t)blockIdx.y * 64 + threadIdx.x], cnt[threadIdx.x]);
}
__global__ void __launch_bounds__(256) k_sort_scatter(Geom g, const DcRec *__restrict__ rec, RecLayout rl, SRec *__restrict__ srec, uint32_t *__restrict__ splits,
                                                      const unsigned *__restrict__ gcnt, unsigned *__restrict__ gcur, int mid_max)
{
  __shared__ unsigned cnt[64], start[64];
  const int ci = blockIdx.y % g.nc, img = blockIdx.y / g.nc;
  const CompGeom &c = g.c[ci];
  const long long nblk = (long long)c.wib * c.hib, b0 = (long long)blockIdx.x * SORT_SLICE;
  if (b0 >= nblk) return;
  const DcRec *r = rec + (size_t)img * rl.per_image + rl.comp_off[ci];
  SRec *p = srec + (size_t)img * rl.per_image + rl.comp_off[ci];
  if (threadIdx.x < 64) cnt[threadIdx.x] = 0;
  __syncthreads();
  const long long b1 = min(nblk, b0 + SORT_SLICE);
  for (long long b = b0 + threadIdx.x; b < b1; b += blockDim.x) atomicAdd(&cnt[63 - min((int)r[b].nz, 63)], 1u);
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned a = 0;
    for (int k = 0; k < 64; k++) { start[k] = a; a += gcnt[(size_t)blockIdx.y * 64 + k]; }
    if (blockIdx.x == 0) {
      splits[4 * blockIdx.y] = start[63 - 32]; splits[4 * blockIdx.y + 1] = start[63 - mid_max]; splits[4 * blockIdx.y + 2] = start[63 - 8];
      splits[4 * blockIdx.y + 3] = (uint32_t)nblk;
    }
  }
  __syncthreads();
  // this slice's range inside every count's run
  if (threadIdx.x < 64) { const unsigned mine = cnt[threadIdx.x]; start[threadIdx.x] += mine ? atomicAdd(&gcur[(size_t)blockIdx.y * 64 + threadIdx.x], mine) : 0u; }
  __syncthreads();
  for (long long b = b0 + threadIdx.x; b < b1; b += blockDim.x) {
    const uint4 q = reinterpret_cast<const uint4 *>(r)[b];        // {norm, raw_dc | nz << 16, mask lo, mask hi}
    const int nz = (int)((q.y >> 16) & 0xFF);
    const unsigned pos = atomicAdd(&start[63 - min(nz, 63)], 1u);
    reinterpret_cast<uint4 *>(p)[pos] = make_uint4(q.x, (unsigned)b, q.z, q.w);
  }
}
static void launch_sort2(const Geom &g, const DcRec *rec, const RecLayout &rl, SRec *srec, uint32_t *splits, unsigned *scratch /* [2][n*nc][64] */, int mid_max, int n, cudaStream_t s)
{
  long long mb = 0;
  for (int ci = 0; ci < g.nc; ci++) mb = max(mb, (long long)g.c[ci].wib * g.c[ci].hib);
  const size_t words = (size_t)n * g.nc * 64;
  cudaMemsetAsync(scratch, 0, 2 * words * sizeof(unsigned), s);
  dim3 grid((unsigned)((mb + SORT_SLICE - 1) / SORT_SLICE), n * g.nc);
  k_sort_count<<<grid, 256, 0, s>>>(g, rec, rl, scratch); LAUNCHED();
  k_sort_scatter<<<grid, 256, 0, s>>>(g, rec, rl, srec, splits, scratch, scratch + words, mid_max); LAUNCHED();
}

// exact int -> float for 0 <= v < 2^23 without the conversion unit
__device__ __forceinline__ float u2f_exact(unsigned v) { return __uint_as_float(0x4B000000u | v) - 8388608.0f; }

// =====================================================================
// AC trellis (third generation; the first two unrolled the entry x predecessor loops over register-resident lists and
// are in the history): rolled loops over shared-memory lists, jcdctmgr.c:1121-1222.  One thread per block, blocks in
// sorted order (k_sort_count / k_sort_scatter), one kernel
// instantiation per count class; the class only sizes the per-thread lists.
//  * phase 1 walks the 63 raw coefficients once (packed fp32x2 conversion / squaring / weighting, scalar prefix chain
//    in the reference's order) and PUSHES an entry {A[p-1], p | raw << 16} for every position p whose plain-quantized
//    value is non-zero -- nothing else of the prefix is kept;
//  * the search runs entry by entry with warp-uniform trip counts: per predecessor s one 8-byte record {-A[p_s], acc_s}
//    and one word {4 p_s | ...} are read, T = (A[i-1] - A[p_s]) + acc_s is formed once and shared by the (up to 3
//    unrolled) candidates, whose distortion is +inf on lanes that do not have them -- so no lane-dependent branch sits
//    inside the predecessor loop; the number of unrolled candidates follows the warp's largest candidate count;
//  * code size is a few hundred instructions (the first two generations unrolled the entry x predecessor loops into
//    5-8 thousand and stalled on instruction fetch), registers ~50, shared memory 12 bytes per list slot and thread.
// =====================================================================
#define T3_THREADS 128
#ifndef SYMREC_DIRECT
#define SYMREC_DIRECT 0
#endif
static_assert(!(SYMREC_DIRECT && SYMREC_SPLIT), "the direct-store A/B aid writes whole 128-byte slots");
// resident CTAs per SM the compiler must allow for the <= 8 entries class, and for the 9..15 entries class.  H100, cfg2:
// 6 (80 registers, no spills) ran the AC stage in 9.84-9.87 ms against 10.06-10.13 at 8 (64 registers, 18 / 20 bytes of
// spill stores / loads); an earlier GPU measured 12 slower than 8
#ifndef T3_MINB_8
#define T3_MINB_8 6
#endif
#ifndef T3_MINB_15
#define T3_MINB_15 6
#endif
#ifndef T3_PRED_UNROLL
#define T3_PRED_UNROLL 4       // predecessor loop: iterations in flight (their shared-memory loads are independent); 1 / 2 / 4: 2.56 / 2.49 / 2.44 ms per 64 4K images
#endif
#define T3_PRAGMA_(x) _Pragma(#x)
#define T3_PRAGMA_UNROLL(n) T3_PRAGMA_(unroll n)
template <int MM> struct T3Smem {
  uint2 rec[MM][T3_THREADS];       // before the entry is processed: {A[p-1], p | raw << 16}; after: {-A[p], accumulated cost}
  unsigned ew[MM][T3_THREADS];     // 4*p | chosen predecessor (1-based entry, 0 = block start) << 8 | chosen value << 16
};

template <int KN>
__device__ __forceinline__ void t3_pred_loop(const int t, const uint2 *__restrict__ rec /* + tid */, const unsigned *__restrict__ ew /* + tid */,
                                             const char *__restrict__ rb, const float before, const float d0, const float d1, const float d2,
                                             float &kb0, int &ks0, float &kb1, int &ks1, float &kb2, int &ks2)
{
T3_PRAGMA_UNROLL(T3_PRED_UNROLL)
  for (int s = 0; s < t; s++) {
    const uint2 r = rec[s * T3_THREADS];
    const int pos4 = (int)(ew[s * T3_THREADS] & 0xFCu);         // (stale words on idle lanes must still give aligned addresses)
    const float T = (before + __uint_as_float(r.x)) + __uint_as_float(r.y);          // :1176
    const char *ra = rb - pos4;
    { const float c = (*reinterpret_cast<const float *>(ra) + d0) + T; if (c < kb0) { kb0 = c; ks0 = s + 1; } }
    if (KN > 1) { const float c = (*reinterpret_cast<const float *>(ra + 256) + d1) + T; if (c < kb1) { kb1 = c; ks1 = s + 1; } }
    if (KN > 2) { const float c = (*reinterpret_cast<const float *>(ra + 512) + d2) + T; if (c < kb2) { kb2 = c; ks2 = s + 1; } }
  }
}
// distortion of candidate value `cand` at a position with divisor q, raw magnitude x (:1149-1151)
__device__ __forceinline__ float t3_dist(const int cand, const int q, const int x, const float lambda, const float wl)
{
  const float fd = u2f_exact((unsigned)abs(cand * q - x));
  return ((fd * fd) * lambda) * wl;
}

template <int MM>
__global__ void __launch_bounds__(T3_THREADS, MM <= 8 ? T3_MINB_8 : MM <= 15 ? T3_MINB_15 : MM <= 32 ? 4 : 2)
k_trellis_ac3(Geom g, const TrellisConsts *__restrict__ tc, const DevHuff *__restrict__ tabs, size_t tabs_set_stride,
              DcRec *__restrict__ rec, RecLayout rl, const SRec *__restrict__ srec, const uint32_t *__restrict__ splits, SymOut so)
{
  const int ci = blockIdx.y % g.nc, img = blockIdx.y / g.nc;
  const CompGeom &c = g.c[ci];
  long long lo, hi;
  {
    const uint4 sp = reinterpret_cast<const uint4 *>(splits)[blockIdx.y];
    if (MM == 64) { lo = 0; hi = sp.x; } else if (MM == 32) { lo = sp.x; hi = sp.y; } else if (MM == 15) { lo = sp.y; hi = sp.z; } else { lo = sp.z; hi = sp.w; }
  }
  const int nchunks = (int)((hi - lo + T3_THREADS - 1) / T3_THREADS);
  if ((int)blockIdx.x >= nchunks) return;
  extern __shared__ __align__(16) unsigned char t3_dyn[];
  T3Smem<MM> &L = *reinterpret_cast<T3Smem<MM> *>(t3_dyn);
  // rate[k][run] (:1163-1175), +inf where the reference skips.  Lanes past their block's last entry run the loops on
  // whatever the lists hold (their results are discarded): such reads stay within 256 bytes in front of the table
  __shared__ __align__(16) float srate_pad[64 + 10 * 64];
  float *srate = srate_pad + 64;
  __shared__ __align__(16) uint4 sEnt[64];                    // per zigzag position {8*Q, reciprocal, weight, -}
  __shared__ __align__(16) float swz[64];
  __shared__ int sqL;
  // final AC symbols of this CTA's blocks (so.hist): run * 10 + size - 1, then EOB, ZRL (sizes are at most 10 where the trellis runs)
  __shared__ unsigned shist[164];
  const int tid = threadIdx.x;
  for (int i = tid; i < 164; i += T3_THREADS) shist[i] = 0;
  uint8_t *acsi = reinterpret_cast<uint8_t *>(t3_dyn);        // table build only
  {
    const DevHuff *ac = reinterpret_cast<const DevHuff *>(reinterpret_cast<const char *>(tabs) + (size_t)blockIdx.y * tabs_set_stride) + (4 + c.ac_tbl);
    for (int i = tid; i < 256; i += T3_THREADS) acsi[i] = ac->size[i];
    const TrellisConsts *tq = qset_of(tc, g, img);             // the image's table set (the other fields are the batch's)
    if (tid < 64) {
      const float w = tq->w_zz[c.qt][tid];
      swz[tid] = w;
      sEnt[tid] = make_uint4((unsigned)tq->q8_zz[c.qt][tid], tq->qmul_zz[c.qt][tid], __float_as_uint(w), 0u);
    }
    if (tid == 0) sqL = tq->qL[c.qt];
  }
  __syncthreads();
  for (int e = tid; e < 640; e += T3_THREADS) {
    const int k = e >> 6, run = e & 63;
    const int zrl = acsi[0xF0], cb = acsi[16 * (run & 15) + k + 1];
    const bool skip = cb == 0 || ((run >> 4) && zrl == 0) || run == 63;
    srate[e] = skip ? __int_as_float(0x7F800000) : (float)(cb + (k + 1) + (run >> 4) * zrl);
  }
  const float eob = (float)acsi[0];
  __syncthreads();                                             // acsi (aliasing the lists) is dead from here on
  const int maxq = (1 << tc->max_coef_bits) - 1;
  const int qL = sqL;
  const size_t rbase = (size_t)img * rl.per_image + rl.comp_off[ci];
  const int use_norm = tc->use_norm;
  const double p1 = tc->p1, p2 = tc->p2; const float lambda_const = tc->lambda_const;
  uint2 *myrec = &L.rec[0][tid]; unsigned *myew = &L.ew[0][tid];
  const char *srate_b = reinterpret_cast<const char *>(srate);
  const float INF = __int_as_float(0x7F800000);

#pragma unroll 1
  for (int chunk = blockIdx.x; chunk < nchunks; chunk += gridDim.x) {
    const long long tix = lo + (long long)chunk * T3_THREADS + tid;
    const bool live = tix < hi;                                // whole warps stay in step (warp reductions below); dead lanes do no memory traffic
    SRec sr; sr.norm = 0.f; sr.lin = 0; sr.nzmask = 0;
    if (live) sr = srec[rbase + tix];
    const unsigned lin = sr.lin;
    const int by = lin / c.wib, bx = lin - by * c.wib;
    const size_t blk = ((size_t)img * c.hpad + by) * c.wpad + bx;
    const int16_t *raw16 = c.raw + blk * 64;
    int16_t *o16 = c.coef + blk * 64;
    uint4 rv[8];
#pragma unroll
    for (int v = 0; v < 8; v++) rv[v] = make_uint4(0, 0, 0, 0);
    // the block's DC value where this kernel will need it (it survives a rewrite of the block; it is the final DC when no
    // DC trellis follows): fetched together with the raw block.  Fetched right in front of the block's stores instead, the
    // kernel ran 3.9x slower wherever blocks are rewritten (progressive profiles: 6.42 vs 1.65 ms per 32 4K images)
    unsigned dc_q = 0;
    const bool want_dc = !so.sym || so.keep_coef || so.dcq_ac;
    if (live) {
      const uint4 *r4 = reinterpret_cast<const uint4 *>(raw16);
#pragma unroll
      for (int v = 0; v < 8; v++) rv[v] = r4[v];
      if (want_dc) dc_q = (unsigned)(unsigned short)o16[0];
    }
    // (the record keeps the norm: the DC trellis derives lambda_dc from it, dc_lambda)
    float lambda;
    {
      const float norm = (float)((double)sr.norm / 63.0);      // :1026-1035
      if (use_norm) lambda = (float)(p1 / (p2 + (double)norm)); else lambda = lambda_const;
    }
    // phase 1: accumulated zero distortion, zigzag order, serial fp32 (:1134); entries pushed where the mask says so
    const unsigned mlo = (unsigned)sr.nzmask, mhi = (unsigned)(sr.nzmask >> 32);
    const int m = __popc(mlo) + __popc(mhi);
    const int mmax = __reduce_max_sync(0xffffffffu, m);
    float azd = 0.0f;
    // (a warp whose 32 blocks have no entry at all -- the tail of the sorted order -- needs neither the prefix nor the search)
    if (mmax != 0) {
      uint2 *push = myrec;
      const float bias = -8421376.0f;   // -(2^23 + 2^15): undoes the exponent trick and the +32768 offset
#pragma unroll
      for (int v = 0; v < 8; v++) {
        const unsigned aw[4] = {rv[v].x, rv[v].y, rv[v].z, rv[v].w};
        const float4 w0 = reinterpret_cast<const float4 *>(swz)[2 * v], w1 = reinterpret_cast<const float4 *>(swz)[2 * v + 1];
        const float ww[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
        const unsigned mw = v < 4 ? mlo : mhi;                   // mask word holding this group's 8 bits
#pragma unroll
        for (int jj = 0; jj < 4; jj++) {
          const unsigned u = aw[jj] ^ 0x80008000u;               // both halves + 32768
          const float fx = __fadd_rn(__uint_as_float(__byte_perm(u, 0x4B000000u, 0x7610)), bias);   // the raw values as floats, exact
          const float fy = __fadd_rn(__uint_as_float(__byte_perm(u, 0x4B000000u, 0x7632)), bias);
          const float2 z = make_float2(__fmul_rn(__fmul_rn(__fmul_rn(fx, fx), lambda), ww[2 * jj]),
                                       __fmul_rn(__fmul_rn(__fmul_rn(fy, fy), lambda), ww[2 * jj + 1]));
          const int i = 8 * v + 2 * jj;
          if (i != 0) {
            // entry word: position | raw value << 16 (one byte permute)
            if (mw & (1u << (i & 31))) { *push = make_uint2(__float_as_uint(azd), __byte_perm(aw[jj], (unsigned)i, 0x1054)); push += T3_THREADS; }
            azd = z.x + azd;
          }
          if (mw & (1u << ((i + 1) & 31))) { *push = make_uint2(__float_as_uint(azd), __byte_perm(aw[jj], (unsigned)(i + 1), 0x3254)); push += T3_THREADS; }
          azd = z.y + azd;
        }
      }
    }
    const float azd63 = azd;
    // phase 2 (:1121-1185): entries in order; all lanes of the warp walk the same entry index.  The end-of-block choice
    // (:1187-1207) rides along: an entry's cost of being the last one is known as soon as the entry is settled.
    int last = 0;
    float best_cost = azd63 + eob;
    // the entry's own constants (fetching them one entry ahead, behind the previous predecessor loop, measured no gain)
    struct Ent { float before, wl, at; int i, rawv, x, q, qv; };
    auto fetch = [&](int t) {
      Ent n;
      const uint2 e = myrec[t * T3_THREADS];
      n.before = __uint_as_float(e.x);                          // A[i-1]
      n.i = (int)(e.y & 63u); n.rawv = (int)e.y >> 16;
      const uint4 en = sEnt[n.i];                               // {8*Q, reciprocal, weight bits, -}
      n.x = abs(n.rawv); n.q = (int)en.x;
      n.wl = __uint_as_float(en.z);
      n.qv = min((int)(__umulhi((unsigned)(n.x + (n.q >> 1)) << 14, en.y) >> qL), maxq);      // :1136-1144
      const float fx = u2f_exact((unsigned)n.x);
      n.at = ((fx * fx) * lambda) * n.wl + n.before;            // A[i], as phase 1 formed it
      return n;
    };
#pragma unroll 1
    for (int t = 0; t < mmax; t++) {
      const bool act = t < m;
      const Ent ce = fetch(t);
      const float before = ce.before, wl = ce.wl, at = ce.at;
      const int i = ce.i, rawv = ce.rawv, x = ce.x, q = ce.q, qv = ce.qv;
      const int nc = act ? nbits_of(qv) : 0;
      const char *rb = srate_b + (i - 1) * 4;                   // rate of run i-1-j at rb[-4j] (+256 per candidate)
      const int ncmax = __reduce_max_sync(0xffffffffu, nc);
      // candidates 0..2 (values 1, 3, 7 below the last one, which is qv itself, :1146-1153); a lane that lacks a candidate
      // gives it an infinite distortion.  Block start as predecessor first: run i-1, zero tail.
      float kb0 = 1e38f, kb1 = 1e38f, kb2 = 1e38f; int ks0 = 0, ks1 = 0, ks2 = 0;
      float best, d0, d1 = INF, d2 = INF; int best_s, best_k;
      d0 = t3_dist(nc > 1 ? 1 : qv, q, x, lambda, wl);
      kb0 = fminf((*reinterpret_cast<const float *>(rb) + d0) + before, kb0);
      if (ncmax <= 1) {
        t3_pred_loop<1>(t, myrec, myew, rb, before, d0, d1, d2, kb0, ks0, kb1, ks1, kb2, ks2);
        best = kb0; best_s = ks0; best_k = kb0 < 1e38f ? 0 : -1;
      } else {
        d1 = nc > 1 ? t3_dist(nc > 2 ? 3 : qv, q, x, lambda, wl) : INF;
        kb1 = fminf((*reinterpret_cast<const float *>(rb + 256) + d1) + before, kb1);
        if (ncmax == 2) t3_pred_loop<2>(t, myrec, myew, rb, before, d0, d1, d2, kb0, ks0, kb1, ks1, kb2, ks2);
        else {
          d2 = nc > 2 ? t3_dist(nc > 3 ? 7 : qv, q, x, lambda, wl) : INF;
          kb2 = fminf((*reinterpret_cast<const float *>(rb + 512) + d2) + before, kb2);
          t3_pred_loop<3>(t, myrec, myew, rb, before, d0, d1, d2, kb0, ks0, kb1, ks1, kb2, ks2);
        }
        // over candidates: smallest cost, ties to the earlier predecessor, then to the earlier candidate (:1157-1184 in its scan order)
        best = 1e38f; best_s = 0; best_k = -1;
        if (kb0 < best) { best = kb0; best_s = ks0; best_k = 0; }
        if (kb1 < best || (kb1 == best && ks1 < best_s)) { best = kb1; best_s = ks1; best_k = 1; }
        if (ncmax > 2 && (kb2 < best || (kb2 == best && ks2 < best_s))) { best = kb2; best_s = ks2; best_k = 2; }
#pragma unroll 1
        for (int k = 3; k < ncmax; k++) {                        // values of 16 and more: rare
          const float dk = k < nc ? t3_dist(k < nc - 1 ? (2 << k) - 1 : qv, q, x, lambda, wl) : INF;
          const char *rk = rb + k * 256;
          float kb = fminf((*reinterpret_cast<const float *>(rk) + dk) + before, 1e38f); int ks = 0;
          float u1 = 1e38f, u2 = 1e38f; int v1 = 0, v2 = 0;
          t3_pred_loop<1>(t, myrec, myew, rk, before, dk, INF, INF, kb, ks, u1, v1, u2, v2);
          if (kb < best || (kb == best && ks < best_s)) { best = kb; best_s = ks; best_k = k; }
        }
      }
      // the value this entry takes if it stays on the chain (:1179, :1143-1153)
      const int cand = (best_k >= 0 && best_k < nc - 1) ? (2 << best_k) - 1 : qv;
      const int sgn = rawv >> 31;
      const int val = (cand ^ sgn) - sgn;
      if (act) {
        myrec[t * T3_THREADS] = make_uint2(__float_as_uint(-at), __float_as_uint(best));
        myew[t * T3_THREADS] = (unsigned)(i << 2) | ((unsigned)best_s << 8) | ((unsigned)val << 16);
        float cst = (best + azd63) - at;
        if (i < 63) cst += eob;
        if (cst < best_cost) { best_cost = cst; last = t + 1; }
      }
    }
    if (live) {
      // output: zeros except the back-tracked chain (:1211-1222)
      uint4 *q4 = reinterpret_cast<uint4 *>(o16);
      auto write_block = [&](int lst) {
        // without want_dc a DC trellis follows and the scans read the DC from dcq: the plane's DC is never read (the
        // DC trellis reads the side records), and on the path where the forward kernel counted the statistics nobody
        // wrote it
        q4[0] = make_uint4(want_dc ? dc_q : 0u, 0, 0, 0);
#pragma unroll
        for (int v = 1; v < 8; v++) q4[v] = make_uint4(0, 0, 0, 0);
        unsigned long long fm = 0;
        while (lst != 0) {
          const unsigned w = myew[(lst - 1) * T3_THREADS];
          const int pos = (int)((w & 0xFFu) >> 2), val = (int)w >> 16;
          o16[pos] = (int16_t)val; if (val) fm |= 1ull << pos;
          lst = (int)((w >> 8) & 0xFFu);
        }
        return fm;
      };
      if (!so.sym) {
        const unsigned long long fm = write_block(last);
        if (SEQ_SPARSE_ENC) rec[rbase + lin].nzmask = fm;
      } else {
        // sequential scans follow: the back-track leaves the block's AC symbols as a record (header word: number of
        // entries, bit 7 = more than SYMREC_SLOTS; entry = symbol | value bits << 16, LAST symbol of the stream first --
        // encode_one_block's order, jchuff.c:600-661, reversed) and counts them for the scan's optimal tables
        // (htest_one_block, jchuff.c:836-878).  The record is put together in this thread's {-A, cost} list, which is
        // dead.  The coefficient block itself is rewritten only if somebody will read it: the debug tap, or the
        // entropy stages when the record overflowed.
        unsigned *scr = reinterpret_cast<unsigned *>(myrec);
        int ns = 0;
#if SYMREC_DIRECT
        unsigned *gout = reinterpret_cast<unsigned *>(so.sym + (rbase + lin) * SYMREC_BYTES);      // A/B: entries straight to global memory
        auto put_sym = [&](unsigned e) { if (ns < SYMREC_SLOTS) gout[ns + 1] = e; ns++; };
#else
        auto put_sym = [&](unsigned e) { if (ns < SYMREC_SLOTS) scr[((ns + 1) >> 1) * (T3_THREADS * 2) + ((ns + 1) & 1)] = e; ns++; };
#endif
        const int last0 = last;
        unsigned w = last ? myew[(last - 1) * T3_THREADS] : 0u;
        if (last == 0 || (w & 0xFCu) != (63u << 2)) { put_sym(0u); if (so.hist) atomicAdd(&shist[160], 1u); }      // EOB
        while (last != 0) {
          const int pos = (int)((w & 0xFFu) >> 2), val = (int)w >> 16;
          const int pr = (int)((w >> 8) & 0xFFu);
          const unsigned wn = pr ? myew[(pr - 1) * T3_THREADS] : 0u;
          const int run = pos - (int)((wn & 0xFFu) >> 2) - 1;
          const int nb = nbits_of(abs(val));
          const unsigned vb = (unsigned)(val + (val >> 31)) & ((1u << nb) - 1u);
          put_sym((unsigned)(((run & 15) << 4) | nb) | vb << 16);
          for (int z = run >> 4; z > 0; z--) put_sym(0xF0u);
          if (so.hist) { atomicAdd(&shist[(run & 15) * 10 + nb - 1], 1u); if (run >> 4) atomicAdd(&shist[161], (unsigned)(run >> 4)); }
          last = pr; w = wn;
        }
#if SYMREC_DIRECT
        gout[0] = ns > SYMREC_SLOTS ? 0x80u : (unsigned)ns; (void)scr;
#else
        scr[0] = ns > SYMREC_SLOTS ? 0x80u : (unsigned)ns;
        // whole 32-byte sectors leave (the words past the last entry are whatever the list held)
        const int nw = 1 + min(ns, SYMREC_SLOTS);
#if SYMREC_SPLIT
        uint4 *dlo = reinterpret_cast<uint4 *>(so.sym + (rbase + lin) * (SYMREC_BYTES / 2));
        uint4 *dhi = reinterpret_cast<uint4 *>(so.sym + (size_t)rl.sym_hi + (rbase + lin) * (SYMREC_BYTES / 2)) - 4;
#else
        uint4 *dlo = reinterpret_cast<uint4 *>(so.sym + (rbase + lin) * SYMREC_BYTES), *dhi = dlo;
#endif
        for (int v = 0; 4 * v < nw; v += 2) {
          const uint2 a = myrec[(2 * v) * T3_THREADS], b = myrec[(2 * v + 1) * T3_THREADS];
          const uint2 c2 = myrec[(2 * v + 2) * T3_THREADS], d2 = myrec[(2 * v + 3) * T3_THREADS];
          uint4 *dst = v < 4 ? dlo : dhi;
          dst[v] = make_uint4(a.x, a.y, b.x, b.y);
          dst[v + 1] = make_uint4(c2.x, c2.y, d2.x, d2.y);
        }
#endif
        if (so.dcq_ac) so.dcq[rbase + lin] = (int16_t)dc_q;          // no DC trellis behind this kernel: the plain-quantized DC is final
        if (so.keep_coef || ns > SYMREC_SLOTS) write_block(last0);
      }
    }
  }
  if (so.hist) {
    __syncthreads();
    uint32_t *gh = so.hist + ((size_t)img * HIST_SLOTS + 4 + c.ac_tbl) * HIST_BINS;
    for (int i = tid; i < 162; i += T3_THREADS) {
      const unsigned v = shist[i];
      if (v) atomicAdd(&gh[i < 160 ? (((i / 10) << 4) | (i % 10 + 1)) : i == 160 ? 0 : 0xF0], v);
    }
  }
}

template <int MM>
static void launch_t3(dim3 grid, cudaStream_t s, const Geom &g, const TrellisConsts *tc, const DevHuff *tabs, size_t tabs_set_stride,
                      DcRec *rec, const RecLayout &rl, const SRec *srec, const uint32_t *splits, const SymOut &so)
{
  // per device: an application may hold encoders on several GPUs in one process, so the opt-in is not cached
  if (sizeof(T3Smem<MM>) + 8192 > 48 * 1024) cudaFuncSetAttribute(k_trellis_ac3<MM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(T3Smem<MM>));
  k_trellis_ac3<MM><<<grid, T3_THREADS, sizeof(T3Smem<MM>), s>>>(g, tc, tabs, tabs_set_stride, rec, rl, srec, splits, so); LAUNCHED();
}
void launch_trellis_sort(const Geom &g, const DcRec *rec, const RecLayout &rl, void *srec, uint32_t *splits, int n, cudaStream_t s)
{
  // splits: 4 words per (image, component), followed by the sort's scratch counters (2 x 64 words each)
  launch_sort2(g, rec, rl, static_cast<SRec *>(srec), splits, splits + (size_t)n * g.nc * 4, 15, n, s);
}
void launch_trellis_ac3(const Geom &g, const TrellisConsts *tc, const DevHuff *tabs, size_t tabs_set_stride,
                        DcRec *rec, const RecLayout &rl, const void *srec, const uint32_t *splits, const SymOut &so, int n, int sms, cudaStream_t s)
{
  long long mb = 0;
  for (int ci = 0; ci < g.nc; ci++) mb = max(mb, (long long)g.c[ci].wib * g.c[ci].hib);
  const unsigned full = (unsigned)((mb + T3_THREADS - 1) / T3_THREADS);
  // CTAs loop over their class's chunks: enough of them per (image, component) to fill the device, few enough to amortise the tables
  unsigned gx = (unsigned)max(1, min((int)full, (sms * 8 * 3 + n * g.nc - 1) / (n * g.nc)));
  dim3 grid(gx, n * g.nc);
  const SRec *sr = static_cast<const SRec *>(srec);
  // largest blocks first: the classes touch disjoint blocks.  The two big-list classes hold 2 / 4 CTAs per SM (96 / 48 KB of
  // lists): a full-size grid of CTAs that mostly find their class empty costs more there than the few chunks are worth,
  // so they get 8 / 16 CTAs per (image, component), still one to two waves when the classes are full (high quality settings)
  launch_t3<64>(dim3(min(gx, 8u), grid.y), s, g, tc, tabs, tabs_set_stride, rec, rl, sr, splits, so);
  launch_t3<32>(dim3(min(gx, 16u), grid.y), s, g, tc, tabs, tabs_set_stride, rec, rl, sr, splits, so);
  launch_t3<15>(grid, s, g, tc, tabs, tabs_set_stride, rec, rl, sr, splits, so);
  launch_t3<8>(grid, s, g, tc, tabs, tabs_set_stride, rec, rl, sr, splits, so);
}

// =====================================================================
// trellis quantization, DC part (jcdctmgr.c:1045-1118 forward, :1308-1327
// back-track).  The Viterbi chain runs along one block row; last_dc carries
// from block row to block row inside an iMCU row (jccoefct.c:418, :1320).
// =====================================================================
// The block's lambda_dc from its record's first word.  Behind k_trellis_ac_band that word holds lambda_dc; behind
// k_trellis_ac3 (from_norm) it still holds the forward kernel's norm, and lambda_dc is derived here with the expression
// of :1026-1035 the AC trellis uses, times the DC weight w0 of the image's table (ac3 does not store it: one scattered
// 4-byte write per block into an array far larger than L2).  tc: lambda fields (the same in every table set).
// (float)((double)f / 63.0) is the correctly rounded fp32 quotient (a double quotient of two floats rounds to float
// without a double-rounding error, 53 >= 2*24 + 2), so one fp32 division gives the same norm for one fp64 division less.
__device__ __forceinline__ float dc_lambda(const float f, const int from_norm, const TrellisConsts *__restrict__ tc, const float w0)
{
  if (!from_norm) return f;
  const float norm = __fdiv_rn(f, 63.0f);
  const float lambda = tc->use_norm ? (float)(tc->p1 / (tc->p2 + (double)norm)) : tc->lambda_const;
  return lambda * w0;
}

// ---------------------------------------------------------------------
// k_trellis_dc_v2: 9 lanes per Viterbi chain (lane k = candidate k), 3 chains
// (iMCU rows) per warp, DC2_WARPS warps per CTA (one where the rows are too
// wide for that many chains' back pointers in shared memory).
//   * the side records of the next 32 blocks are fetched by the whole warp
//     (coalesced) while the current 32 are processed from shared memory;
//   * everything that does not depend on the Viterbi state -- candidate values,
//     distortions and the 9 rate terms (float)(bits + size[bits]) + dist of the
//     step -- is computed ahead of the 9 shuffles that bring the predecessors'
//     accumulated costs, so the state-dependent part of a step is 9 adds and a
//     4-level first-minimum tree;
//   * the serial back-track only chases one byte per block through shared
//     memory; candidates are turned into coefficients by all 32 lanes afterwards.
// Arithmetic, association order and tie-breaks are those of quantize_trellis.
// ---------------------------------------------------------------------
#ifndef DC2_WARPS
#define DC2_WARPS 2
#endif
// FAST instantiation: the rates of a step's 9 predecessor differences, |D0 -+ l|, come from one table indexed by the
// signed difference (consecutive words from one base address) instead of abs / find-leading-one / table per difference
#define DC_TAB_HALF 512
// FLO: index of the most significant set bit, 0xFFFFFFFF for 0, so that
// nbits(v) == bfind(v) + 1 (JPEG_NBITS) without the clz arithmetic.
__device__ __forceinline__ int bfind_u32(unsigned v) { int r; asm("bfind.u32 %0, %1;" : "=r"(r) : "r"(v)); return r; }

// FAST: 9 candidates and no clamping possible for any DC value (lim - 1 >= the
// largest reachable candidate): the 81 candidate differences of a step collapse
// to D0 - psgn*l, and no candidate needs masking.
// VERT: trellis_delta_dc_weight > 0 (cjpeg -trellis-dc-ver-weight): from an iMCU row's second block row on, a candidate's
// distortion is blended with the difference of vertical gradients to the finished block above (:1069-1086).
template <bool FAST, bool VERT>
__global__ void __launch_bounds__(DC2_WARPS * 32) k_trellis_dc_v2(Geom g, const TrellisConsts *__restrict__ tc,
                                                                 const DevHuff *__restrict__ tabs, size_t tabs_set_stride,
                                                                 const DcRec *__restrict__ rec, RecLayout rl, int max_wib, int16_t *__restrict__ dcq, int write_coef,
                                                                 int lambda_from_norm)
{
  extern __shared__ __align__(16) unsigned char dsm[];
  __shared__ float T[36];                                   // T[1 + bfind(|d|)] = (float)(bits + ehufsi[bits])
  __shared__ float Tt[FAST ? 2 * DC_TAB_HALF + 8 : 1];      // Tt[d + DC_TAB_HALF] = T[1 + bfind(|d|)], -DC_TAB_HALF <= d < DC_TAB_HALF + 8
  __shared__ int4 stage[DC2_WARPS][3][32];                  // per staged block {|raw DC|, qval - half, +1 / -1, lambda bits}: what a step needs of the record
  __shared__ int2 vstage[DC2_WARPS][3][32];                 // VERT: per staged block {raw DC above - raw DC, final DC above * q}
  const int ci = blockIdx.y % g.nc, img = blockIdx.y / g.nc;
  const CompGeom &c = g.c[ci];
  // the tables are filled in strides of DC2_WARPS * 32 entries, a one-warp CTA's threads taking two slots each (with a
  // stride of blockDim.x the FAST kernel needs one register more)
  {
    const DevHuff *dc = reinterpret_cast<const DevHuff *>(reinterpret_cast<const char *>(tabs) + (size_t)blockIdx.y * tabs_set_stride) + c.dc_tbl;
    for (int t = threadIdx.x; t < DC2_WARPS * 32; t += blockDim.x)
      for (int i = t; i < 33; i += DC2_WARPS * 32) T[i] = (float)(i + (int)dc->size[i]);
  }
  __syncthreads();
  if (FAST) {
    for (int t = threadIdx.x; t < DC2_WARPS * 32; t += blockDim.x)
      for (int i = t; i < 2 * DC_TAB_HALF + 8; i += DC2_WARPS * 32) Tt[i] = T[1 + bfind_u32((unsigned)abs(i - DC_TAB_HALF))];
    __syncthreads();
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int grp = lane / 9, k = lane - grp * 9;                 // lanes 27..31: grp == 3 (help with loads only)
  const int gsel = grp < 3 ? grp : 0;
  const int gbase = gsel * 9;
  const int n_imcu = (c.hib + c.v - 1) / c.v;
  const int imcu0 = (blockIdx.x * (blockDim.x >> 5) + warp) * 3; // first of this warp's three chains
  const int wib = c.wib;
  // back pointers: 9 nibbles per block packed into 5 bytes (candidates 2i, 2i+1 in byte i; byte 4 = candidate 8 in the
  // low nibble, and after the back-track the block's chosen candidate in the high nibble)
  uint8_t *btw = dsm + (size_t)warp * 3 * max_wib * 5;          // [3][max_wib][5]
  uint8_t *bt = btw + (size_t)gsel * max_wib * 5;
  tc = qset_of(tc, g, img);
  const int q = tc->q8_zz[c.qt][0];
  const float w0 = tc->w_zz[c.qt][0];
  int ncand = (2 + 60 / (q >> 3)) | 1; if (ncand > 9) ncand = 9;     // get_num_dc_trellis_candidates (:929-933)
  const int half = ncand / 2;
  const int lim = 1 << tc->max_coef_bits;
  const float INF = __int_as_float(0x7f800000);
  const size_t comp_rec = (size_t)img * rl.per_image + rl.comp_off[ci];
  const int qhalf = q / 2;
  const unsigned qmul = tc->dc_mul[c.qt]; const int qshift = tc->dc_shift[c.qt];
  const float vweight = tc->delta_dc_weight;
  // a block's final DC from its raw DC and its chosen candidate j
  auto final_dc = [&](const int raw, const int j) {
    int v = (int)(((unsigned long long)(unsigned)(abs(raw) + qhalf) * qmul) >> qshift) - half + j;
    if (v >= lim) v = lim - 1;
    if (v <= -lim) v = -lim + 1;
    return raw < 0 ? -v : v;
  };
  int last_dc = 0;                                                // per chain (uniform inside a 9-lane group)
  for (int br = 0; br < c.v; br++) {
    const bool vert = VERT && br > 0;
    // rows of the three chains; a chain without this row idles on row 0 of the component
    int rowg[3]; bool okg[3];
#pragma unroll
    for (int gg = 0; gg < 3; gg++) { int r = (imcu0 + gg) * c.v + br; okg[gg] = (imcu0 + gg) < n_imcu && r < c.hib; rowg[gg] = okg[gg] ? r : 0; }
    const bool rowok = grp < 3 && okg[gsel];
    DcRec nxt[3]; int up[3];                                      // up: raw DC of the block above (vert)
#pragma unroll
    for (int gg = 0; gg < 3; gg++) {
      nxt[gg] = rec[comp_rec + (size_t)rowg[gg] * wib + min(lane, wib - 1)];
      if (vert) up[gg] = rec[comp_rec + (size_t)max(rowg[gg] - 1, 0) * wib + min(lane, wib - 1)].raw_dc;
    }
    float acc = 0.f;
    // previous block's candidate l is psgn * clamp(pbase + l); for the row's first block every
    // predecessor is last_dc with zero accumulated cost (pstep = 0)
    int pbase = last_dc, psgn = 1, pstep = 0;
    uint8_t *btp = bt + (k >> 1);
    for (int bi0 = 0; bi0 < wib; bi0 += 32) {
      __syncwarp();
#pragma unroll
      for (int gg = 0; gg < 3; gg++) {
        const int raw = nxt[gg].raw_dc, x = abs(raw);
        const int qval = (int)(((unsigned long long)(unsigned)(x + qhalf) * qmul) >> qshift);       // (x + q/2) / q, exact
        stage[warp][gg][lane] = make_int4(x, qval - half, 1 + 2 * (raw >> 31), __float_as_int(dc_lambda(nxt[gg].lambda_dc, lambda_from_norm, tc, w0)));
        // the block above still has the candidate the last back-track chose in its back-pointer entry: this row's steps
        // overwrite an entry only when they reach its block
        if (vert) vstage[warp][gg][lane] = make_int2(up[gg] - raw, final_dc(up[gg], btw[((size_t)gg * max_wib + min(bi0 + lane, wib - 1)) * 5 + 4] >> 4) * q);
      }
      __syncwarp();
      if (bi0 + 32 < wib) {
#pragma unroll
        for (int gg = 0; gg < 3; gg++) {
          nxt[gg] = rec[comp_rec + (size_t)rowg[gg] * wib + min(bi0 + 32 + lane, wib - 1)];
          if (vert) up[gg] = rec[comp_rec + (size_t)max(rowg[gg] - 1, 0) * wib + min(bi0 + 32 + lane, wib - 1)].raw_dc;
        }
      }
      const int nstep = min(32, wib - bi0);
      const int4 *sp = &stage[warp][gsel][0];
      const int2 *vp = &vstage[warp][gsel][0];
#pragma unroll 1
      for (int st = 0; st < nstep; st++) {
        const int4 r = sp[st];
        const int x = r.x, base = r.y, sgn = r.z;                   // |raw DC|, qval - half, sign
        int cd = base + k;
        if (!FAST) { if (cd >= lim) cd = lim - 1; if (cd <= -lim) cd = -lim + 1; }
        const int delta = cd * q - x;
        float dist = (float)(delta * delta) * __int_as_float(r.w);
        cd *= sgn;
        if (vert) {
          const int2 v = vp[st];
          const int d2 = v.x - (v.y - cd * q);
          const float vd = (float)(d2 * d2) * __int_as_float(r.w);
          dist += vweight * (vd - dist);
        }
        // rate + distortion against every predecessor candidate l (independent of the Viterbi state)
        float rd[9];
        if (FAST) {
          const int D0 = cd - psgn * pbase, dstep = -psgn * pstep;
          // |D0 + dstep l| = |E0 + l| with E0 = -+D0 when dstep = -+1 (every block but a row's first)
          const int E0 = dstep < 0 ? -D0 : D0;
          if (__all_sync(0xffffffffu, pstep != 0 && (unsigned)(E0 + DC_TAB_HALF) < (unsigned)(2 * DC_TAB_HALF))) {
            const float *tp = Tt + (E0 + DC_TAB_HALF);
#pragma unroll
            for (int l = 0; l < 9; l++) rd[l] = tp[l] + dist;
          } else {
#pragma unroll
            for (int l = 0; l < 9; l++) rd[l] = T[1 + bfind_u32((unsigned)abs(D0 + dstep * l))] + dist;
          }
        } else {
#pragma unroll
          for (int l = 0; l < 9; l++) {
            int v = pbase + pstep * l;
            if (pstep) { if (v >= lim) v = lim - 1; if (v <= -lim) v = -lim + 1; }
            rd[l] = T[1 + bfind_u32((unsigned)abs(cd - psgn * v))] + dist;
          }
        }
        // state-dependent part: predecessors' accumulated costs, first minimum (strict '<', ascending l)
        float cst[9];
#pragma unroll
        for (int l = 0; l < 9; l++) {
          float pa = __shfl_sync(0xffffffffu, acc, gbase + l);
          cst[l] = (FAST || l < ncand) ? rd[l] + pa : INF;
        }
        float c01 = cst[0]; int i01 = 0; if (cst[1] < c01) { c01 = cst[1]; i01 = 1; }
        float c23 = cst[2]; int i23 = 2; if (cst[3] < c23) { c23 = cst[3]; i23 = 3; }
        float c45 = cst[4]; int i45 = 4; if (cst[5] < c45) { c45 = cst[5]; i45 = 5; }
        float c67 = cst[6]; int i67 = 6; if (cst[7] < c67) { c67 = cst[7]; i67 = 7; }
        if (c23 < c01) { c01 = c23; i01 = i23; }
        if (c67 < c45) { c45 = c67; i45 = i67; }
        if (c45 < c01) { c01 = c45; i01 = i45; }
        if (cst[8] < c01) { c01 = cst[8]; i01 = 8; }
        acc = (FAST || k < ncand) ? c01 : INF;
        {
          const int hi = __shfl_down_sync(0xffffffffu, i01, 1);          // candidate k+1's pointer (lane k+1 of the same chain for even k < 8)
          const int nib = (FAST || k < ncand) ? i01 : 0, nibhi = (k < 8 && (FAST || k + 1 < ncand)) ? hi : 0;
          if (rowok && !(k & 1)) *btp = (uint8_t)(nib | (nibhi << 4));
        }
        btp += 5;
        pbase = base; psgn = sgn; pstep = 1;
      }
    }
    // first minimum over the candidates (:1309-1313)
    int j = 0; float bj = __shfl_sync(0xffffffffu, acc, gbase);
#pragma unroll
    for (int i = 1; i < 9; i++) { float a = __shfl_sync(0xffffffffu, acc, gbase + i); if (i < ncand && a < bj) { bj = a; j = i; } }
    __syncwarp();
    // serial back-track: chosen candidate of block bi goes to bt[bi][0]
    if (rowok && k == 0) {
#pragma unroll 4
      for (int bi = wib - 1; bi >= 0; bi--) {
        uint8_t *bb = bt + (size_t)bi * 5;
        const int byte = bb[j >> 1];
        const int jn = (j & 1) ? (byte >> 4) : (byte & 15);
        bb[4] = (uint8_t)((bb[4] & 15) | (j << 4));
        j = jn;
      }
    }
    __syncwarp();
    // candidates -> coefficients, all lanes; the row's last value seeds the next row (jccoefct.c:418, :1320)
#pragma unroll
    for (int gg = 0; gg < 3; gg++) {
      const uint8_t *btg = btw + (size_t)gg * max_wib * 5;
      int lastv = 0;
      for (int bi = lane; bi < wib && okg[gg]; bi += 32) {
        const int cdv = final_dc(rec[comp_rec + (size_t)rowg[gg] * wib + bi].raw_dc, btg[(size_t)bi * 5 + 4] >> 4);
        if (write_coef) c.coef[(((size_t)img * c.hpad + rowg[gg]) * c.wpad + bi) * 64] = (int16_t)cdv;
        if (dcq) dcq[comp_rec + (size_t)rowg[gg] * wib + bi] = (int16_t)cdv;
        if (bi == wib - 1) lastv = cdv;
      }
      lastv = __shfl_sync(0xffffffffu, lastv, (wib - 1) & 31);
      if (grp == gg) last_dc = lastv;
    }
    __syncwarp();
  }
}

void launch_trellis_dc(const Geom &g, const TrellisConsts *tc, const DevHuff *tabs, size_t tabs_set_stride,
                       const DcRec *rec, const RecLayout &rl, int vertical, int dc_fast, int16_t *dcq, int write_coef,
                       int lambda_from_norm, int n, cudaStream_t s)
{
  int n_imcu = 0, max_wib = 0;
  for (int ci = 0; ci < g.nc; ci++) { n_imcu = max(n_imcu, (g.c[ci].hib + g.c[ci].v - 1) / g.c[ci].v); max_wib = max(max_wib, g.c[ci].wib); }
  // 5 bytes of back pointers per block for each of a warp's 3 chains: DC2_WARPS warps per CTA up to 200 KB, one warp for
  // wider rows (8188 blocks, 65500 samples, take 122 820 bytes)
  int warps = DC2_WARPS;
  size_t smem = (size_t)warps * 3 * max_wib * 5;
  if (smem > 200 * 1024) { warps = 1; smem = (size_t)3 * max_wib * 5; }
  auto kern = vertical ? (dc_fast ? k_trellis_dc_v2<true, true> : k_trellis_dc_v2<false, true>)
                       : (dc_fast ? k_trellis_dc_v2<true, false> : k_trellis_dc_v2<false, false>);
  // beyond 48 KB with the kernel's static shared memory (under 9 KB); per device, so not cached: encoders on several
  // GPUs may live in one process
  if (smem + 9 * 1024 > 48 * 1024) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  dim3 grid((n_imcu + warps * 3 - 1) / (warps * 3), n * g.nc);
  // the DC quantizer comes from each image's table set (TrellisConsts.dc_mul / dc_shift)
  kern<<<grid, warps * 32, smem, s>>>(g, tc, tabs, tabs_set_stride, rec, rl, max_wib, dcq, write_coef || !dcq, lambda_from_norm);
  LAUNCHED();
}

// =====================================================================
// entropy coding, pass A: bits per block; pass B: exclusive scan;
// pass C: bit packing; pass D: 0xFF byte stuffing + end-of-scan padding.
// (encode_mcu_huff/encode_one_block jchuff.c:563-763, flush_bits :479-533)
// =====================================================================
struct ScanTables {            // the 8 table slots of one image, staged in shared memory
  uint16_t code[HIST_SLOTS][256];
  uint8_t size[HIST_SLOTS][256];
};
__device__ __forceinline__ void load_scan_tables(ScanTables &st, const DevHuff *tabs, size_t stride, int img, const Geom &g, const ScanDesc &sd, bool want_codes)
{
  const DevHuff *t = reinterpret_cast<const DevHuff *>(reinterpret_cast<const char *>(tabs) + (size_t)img * stride);
  for (int i = 0; i < sd.ncomps; i++) {
    const CompGeom &c = g.c[sd.ci[i]];
    int slots[2] = {c.dc_tbl, 4 + c.ac_tbl};
    for (int z = 0; z < 2; z++) {
      int sl = slots[z];
      for (int k = threadIdx.x; k < 256; k += blockDim.x) { st.size[sl][k] = t[sl].size[k]; if (want_codes) st.code[sl][k] = t[sl].code[k]; }
    }
  }
}

struct CountSink {
  const uint8_t *dsz, *asz; unsigned bits; int bad;
  __device__ void dc(int nb, int) { int s = dsz[nb]; if (!s) bad = 1; bits += s + nb; }
  __device__ void ac(int sym, int nb, int) { int s = asz[sym]; if (!s) bad = 1; bits += s + nb; }
};

// sum of v over the CTA (256 threads), result valid in thread 0
__device__ __forceinline__ unsigned cta_sum_256(unsigned v, unsigned *ws /* [8] shared */)
{
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = v;
  __syncthreads();
  unsigned r = 0;
  if (threadIdx.x == 0) for (int i = 0; i < 8; i++) r += ws[i];
  return r;
}

// exclusive prefix of v inside the CTA (256 threads) and the CTA total (valid in all threads)
__device__ __forceinline__ unsigned cta_excl_scan_256(unsigned v, unsigned *ws /* [9] shared */, unsigned &total)
{
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  unsigned x = v;
  for (int o = 1; o < 32; o <<= 1) { unsigned y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
  if (lane == 31) ws[wid] = x;
  __syncthreads();
  unsigned before = 0, tot = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) { unsigned w = ws[i]; if (i < wid) before += w; tot += w; }
  total = tot;
  return before + x - v;
}

// One tile = the 256 blocks of one CTA; tile_bits[img][tile] = bits the tile emits; blk_bits[img][t] = bits
// the tile's blocks before t emit (exclusive prefix inside the tile).
__global__ void __launch_bounds__(256) k_block_bits_seq(Geom g, ScanDesc sd, const DcRec *__restrict__ nz_rec, const uint8_t *__restrict__ sym, const int16_t *__restrict__ dcq,
                                                        RecLayout rl, const DevHuff *__restrict__ tabs, size_t stride,
                                                        uint32_t *__restrict__ blk_bits, uint32_t *__restrict__ tile_bits, uint32_t *__restrict__ status)
{
  __shared__ ScanTables st;
  __shared__ unsigned ws[8];
  int img = blockIdx.y;
  load_scan_tables(st, tabs, stride, img, g, sd, false);
  __syncthreads();
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  unsigned bits = 0;
  if (t < sd.nblocks && sym) {
    const CompGeom &c = g.c[sd.ci[sd.k_comp[(int)(t % sd.bim)]]];
    CountSink sink{st.size[c.dc_tbl], st.size[4 + c.ac_tbl], 0u, 0};
    walk_seq_rec(g, sd, sym, dcq, rl, img, t, sink);
    if (sink.bad) atomicOr(&status[img], 2u);
    bits = sink.bits;
  } else if (t < sd.nblocks) {
    int sci, k; long long mcu;
    const int16_t *blk = block_ptr(g, sd, img, t, sci, mcu, k);
    int last = prev_dc(g, sd, img, t, sci, mcu, k);
    const CompGeom &c = g.c[sd.ci[sci]];
    CountSink sink{st.size[c.dc_tbl], st.size[4 + c.ac_tbl], 0u, 0};
    if (SEQ_SPARSE_STATS && nz_rec) walk_seq_sparse(blk, block_nzmask(g, sd, nz_rec, rl, img, sci, mcu, k), last, sink);
    else walk_seq_block(blk, last, sink);
    if (sink.bad) atomicOr(&status[img], 2u);
    bits = sink.bits;
  }
  unsigned tot;
  const unsigned pre = cta_excl_scan_256(bits, ws, tot);
  if (t < sd.nblocks) blk_bits[(size_t)img * sd.nblocks + t] = pre;
  if (threadIdx.x == 0) tile_bits[(size_t)img * gridDim.x + blockIdx.x] = tot;
}

struct BitSink {
  uint32_t *buf; unsigned long long widx; unsigned long long acc; int nacc;
  const uint16_t *dco, *aco; const uint8_t *dsz, *asz;
  __device__ void put(unsigned code, int size) {
    acc = (acc << size) | (code & ((1u << size) - 1u)); nacc += size;
    if (nacc >= 32) { unsigned w = (unsigned)(acc >> (nacc - 32)); if (w) atomicOr(&buf[widx], w); widx++; nacc -= 32; }
  }
  __device__ void dc(int nb, int v) { put(dco[nb], dsz[nb]); if (nb) put((unsigned)v, nb); }
  __device__ void ac(int sym, int nb, int v) { put(aco[sym], asz[sym]); if (nb) put((unsigned)v, nb); }
  __device__ void finish() { if (nacc > 0) { unsigned w = (unsigned)(acc << (32 - nacc)); if (w) atomicOr(&buf[widx], w); } }
};

// Scan layout, one CTA per image:
//   tile_base[img][tile] = bits emitted before the tile (exclusive scan of tile_bits);
//   with a restart interval (sd.ri MCUs), every segment but the last is padded to a byte boundary and
//   followed by the 16 bits of its RSTn marker (emit_restart, jchuff.c:668-686): seg_corr[img][s] = padding +
//   marker bits inserted before segment s;
//   total_bits[img] = bits of the whole unstuffed scan; flags an output buffer that is too small.
__device__ __forceinline__ unsigned long long bits_before(const unsigned long long *tb, const uint32_t *pre, long long nblocks, long long t, unsigned long long total)
{
  return t < nblocks ? tb[t >> 8] + pre[t] : total;
}
__global__ void __launch_bounds__(256) k_scan_layout(ScanDesc sd, const uint32_t *__restrict__ blk_bits, const uint32_t *__restrict__ tile_bits,
                                                     int ntiles, unsigned long long *__restrict__ tile_base, uint32_t *__restrict__ seg_corr,
                                                     long long seg_stride, unsigned long long *__restrict__ total_bits,
                                                     size_t capacity_bits, uint32_t *__restrict__ status)
{
  __shared__ unsigned ws[9];
  __shared__ unsigned long long carry;
  const int img = blockIdx.x;
  const uint32_t *tbits = tile_bits + (size_t)img * ntiles;
  unsigned long long *tb = tile_base + (size_t)img * ntiles;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < ntiles; base += 256) {
    const int i = base + threadIdx.x;
    unsigned v = i < ntiles ? tbits[i] : 0u, tot;
    unsigned pre = cta_excl_scan_256(v, ws, tot);
    if (i < ntiles) tb[i] = carry + pre;
    __syncthreads();
    if (threadIdx.x == 0) carry += tot;
    __syncthreads();
  }
  const unsigned long long total = carry;
  unsigned long long grand = total;
  if (sd.ri) {
    const uint32_t *pre = blk_bits + (size_t)img * sd.nblocks;
    uint32_t *sc = seg_corr + (size_t)img * seg_stride;
    const long long seglen = (long long)sd.ri * sd.bim, nseg = (sd.nblocks + seglen - 1) / seglen;
    __syncthreads();
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (long long base = 0; base < nseg; base += 256) {
      const long long sgi = base + threadIdx.x;
      unsigned pad = 0, tot;
      if (sgi < nseg - 1) {
        unsigned long long a = bits_before(tb, pre, sd.nblocks, (sgi + 1) * seglen, total) - bits_before(tb, pre, sd.nblocks, sgi * seglen, total);
        pad = (unsigned)((8 - (a & 7)) & 7) + 16;
      }
      unsigned before = cta_excl_scan_256(pad, ws, tot);
      if (sgi < nseg) sc[sgi] = (uint32_t)(carry + before);
      __syncthreads();
      if (threadIdx.x == 0) carry += tot;
      __syncthreads();
    }
    grand = total + carry;
  }
  if (threadIdx.x == 0) {
    total_bits[img] = grand;
    if (grand + 64 > capacity_bits || grand >= (1ull << 32)) atomicOr(&status[img], 4u);    // does not fit: host retries with a larger buffer
  }
}

// end of a restart segment (not the scan's last): 1-bits up to the byte boundary, then RSTn, whose 0xFF
// must not be byte-stuffed: its position is recorded in the marker bitmap (one bit per unstuffed byte)
__device__ __forceinline__ void emit_restart_marker(BitSink &sink, const ScanDesc &sd, long long t, uint32_t *__restrict__ mark)
{
  const long long seglen = (long long)sd.ri * sd.bim;
  if ((t + 1) % seglen != 0 || t + 1 >= sd.nblocks) return;
  const unsigned long long pos = sink.widx * 32ull + (unsigned)sink.nacc;
  const int pad = (int)((8 - (pos & 7)) & 7);
  if (pad) sink.put((1u << pad) - 1u, pad);
  const unsigned long long byte = (pos + pad) >> 3;
  sink.put(0xFFD0u + (unsigned)((t / seglen) & 7), 16);
  atomicOr(&mark[byte >> 5], 1u << (byte & 31));
}

// the sequential packer's AC symbols: code and size from one table word, code and value bits in one put (at most 16 + 14 bits)
struct BitSinkQ : BitSink {
  const uint32_t *acs;          // code | size << 16
  __device__ void ac(int sym, int nb, int v) { const unsigned e = acs[sym]; put(((e & 0xFFFFu) << nb) | ((unsigned)v & ((1u << nb) - 1u)), (int)(e >> 16) + nb); }
};

__global__ void __launch_bounds__(256) k_encode_seq(Geom g, ScanDesc sd, const DcRec *__restrict__ rec, const uint8_t *__restrict__ sym, const int16_t *__restrict__ dcq,
                                                    RecLayout rl, const DevHuff *__restrict__ tabs, size_t stride,
                                                    const uint32_t *__restrict__ blk_bits, const uint32_t *__restrict__ tile_bits /* per-tile totals: not read here */,
                                                    const unsigned long long *__restrict__ tile_base,
                                                    const uint32_t *__restrict__ seg_corr, long long seg_stride,
                                                    uint32_t *__restrict__ bitbuf, size_t bitbuf_stride_words,
                                                    uint32_t *__restrict__ mark, size_t mark_stride_words, const uint32_t *__restrict__ status)
{
  __shared__ ScanTables st;
  __shared__ uint32_t acs[4][256];
  int img = blockIdx.y;
  load_scan_tables(st, tabs, stride, img, g, sd, true);
  __syncthreads();
  for (int i = 0; i < sd.ncomps; i++) {
    const int sl = g.c[sd.ci[i]].ac_tbl;
    for (int k = threadIdx.x; k < 256; k += blockDim.x) acs[sl][k] = (uint32_t)st.code[4 + sl][k] | (uint32_t)st.size[4 + sl][k] << 16;
  }
  __syncthreads();
  if (status[img] & ~1u) return;            // an earlier stage flagged this image (overflow / bad coefficient)
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned long long tb = tile_base[(size_t)img * gridDim.x + blockIdx.x];
  uint32_t *gbuf = bitbuf + (size_t)img * bitbuf_stride_words;
  if (t < sd.nblocks) {
    unsigned long long off = tb + blk_bits[(size_t)img * sd.nblocks + t];
    if (sd.ri) off += seg_corr[(size_t)img * seg_stride + t / ((long long)sd.ri * sd.bim)];
    const CompGeom &c = g.c[sd.ci[sd.k_comp[(int)(t % sd.bim)]]];
    BitSinkQ sink;
    sink.buf = gbuf; sink.widx = off >> 5; sink.acc = 0; sink.nacc = (int)(off & 31);
    sink.dco = st.code[c.dc_tbl]; sink.aco = st.code[4 + c.ac_tbl]; sink.dsz = st.size[c.dc_tbl]; sink.asz = st.size[4 + c.ac_tbl];
    sink.acs = acs[c.ac_tbl];
    if (sym) walk_seq_rec(g, sd, sym, dcq, rl, img, t, sink);
    else {
      int sci, k; long long mcu;
      const int16_t *blk = block_ptr(g, sd, img, t, sci, mcu, k);
      int last = prev_dc(g, sd, img, t, sci, mcu, k);
      if (SEQ_SPARSE_ENC && rec) walk_seq_sparse(blk, block_nzmask(g, sd, rec, rl, img, sci, mcu, k), last, sink);
      else walk_seq_block(blk, last, sink);
    }
    if (sd.ri) emit_restart_marker(sink, sd, t, mark + (size_t)img * mark_stride_words);
    sink.finish();
  }
}

// ---------------------------------------------------------------------
// Single-pass scan with decoupled look-back (Merrill & Garland, "Single-pass Parallel Prefix Scan with Decoupled
// Look-back", NVIDIA 2016) for the stuffer's output offsets.  A CTA takes its tile from a per-(launch, image) ticket, so
// it only ever waits for tiles that started before it, and every tile that can be a predecessor publishes its
// descriptor whatever the image's status says: the waits end by construction.
// Descriptor (64-bit, written with st.release, read with ld.acquire): bits 62..63 flag (0 not yet, 1 aggregate: the
// tile's own count, 2 inclusive: the count of the tile and all before it), bits 0..61 the value.
// ---------------------------------------------------------------------
#define LB_AGG (1ull << 62)
#define LB_INC (2ull << 62)
__device__ __forceinline__ void lb_publish(unsigned long long *d, unsigned long long v)
{
  asm volatile("st.release.gpu.global.u64 [%0], %1;" :: "l"(d), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long lb_peek(const unsigned long long *d)
{
  unsigned long long v;
  asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(d) : "memory");
  return v;
}
// sum of the values of the tiles before `tile` (> 0) of the descriptor array desc, called by a whole warp: the lanes read
// 32 predecessors' descriptors at a time (waiting until all have published), add the aggregates after the nearest
// inclusive one, and step back 32 tiles when there is none.  Every predecessor holds an earlier ticket, is running or
// done, and publishes without waiting on anything, so the spin ends.
__device__ __forceinline__ unsigned long long lb_lookback(const unsigned long long *desc, int tile)
{
  const int lane = threadIdx.x & 31;
  unsigned long long sum = 0;
  for (int j_end = tile;; j_end -= 32) {
    const int j = j_end - 32 + lane;
    unsigned long long d = LB_INC;                            // before tile 0: never chosen, tile 0 is inclusive
    if (j >= 0) while (!((d = lb_peek(desc + j)) >> 62)) __nanosleep(32);
    const unsigned inc = __ballot_sync(0xffffffffu, (d >> 62) == 2);
    const int hi = inc ? 31 - __clz(inc) : -1;                // nearest inclusive predecessor in the window
    unsigned long long v = lane >= hi ? d & ((1ull << 62) - 1) : 0ull;
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    sum += v;
    if (inc) return sum;
  }
}

// ---------------------------------------------------------------------
// byte stuffing (jchuff.c:386-435 emit byte / 0xFF00) + final 1-bit padding (flush_bits: 7 one-bits, then drop the
// partial byte), in one pass.  A tile is STUFF_TILE_WORDS words = 4096 stream bytes, one CTA: it counts its 0xFF bytes
// (not the restart markers'), publishes that count at once, takes its output offset from the look-back, stages its
// stuffed bytes (at most 8 KB) in shared memory at the output's 16-byte phase and stores them with 16-byte stores (byte
// stores only at its two ends: neighbouring tiles write disjoint bytes).  The tile holding the last stream byte
// publishes the scan size and the next scan's start.
// ---------------------------------------------------------------------
#define STUFF_THREADS 256
#define STUFF_TILE_WORDS (STUFF_THREADS * 4)
__device__ __forceinline__ uint4 stuff_load(const uint32_t *__restrict__ src, unsigned long long nbytes, unsigned padbits,
                                            unsigned long long w0, int &nb)
{
  // 4 words = 16 stream bytes starting at word w0; nb = valid bytes among them; pad the last byte with 1-bits
  uint4 q = make_uint4(0, 0, 0, 0);
  nb = 0;
  if (w0 * 4 < nbytes) {
    unsigned long long rem = nbytes - w0 * 4;
    nb = rem >= 16 ? 16 : (int)rem;
    q = *reinterpret_cast<const uint4 *>(src + w0);
    if (rem <= 16 && padbits) {
      unsigned m = ((1u << padbits) - 1u) << (8 * (3 - ((nb - 1) & 3)));
      int wi = (nb - 1) >> 2;
      if (wi == 0) q.x |= m; else if (wi == 1) q.y |= m; else if (wi == 2) q.z |= m; else q.w |= m;
    }
  }
  return q;
}
// 16 bits of the marker bitmap for the 16 stream bytes starting at word w0 (w0 % 4 == 0): bit j = byte j is the
// 0xFF of a restart marker and must not be stuffed
__device__ __forceinline__ unsigned marker_bits16(const uint32_t *__restrict__ mark, unsigned long long w0)
{
  if (!mark) return 0u;
  const unsigned long long byte0 = w0 * 4;
  return (mark[byte0 >> 5] >> (byte0 & 31)) & 0xFFFFu;
}
__device__ __forceinline__ unsigned count_ff16(uint4 q, int nb, unsigned mk)
{
  unsigned w[4] = {q.x, q.y, q.z, q.w}; unsigned c = 0;
#pragma unroll
  for (int j = 0; j < 16; j++) c += (j < nb) && (((w[j >> 2] >> (24 - 8 * (j & 3))) & 0xFF) == 0xFF) && !((mk >> j) & 1u);
  return c;
}
__global__ void __launch_bounds__(STUFF_THREADS) k_stuff(const uint32_t *__restrict__ bitbuf, size_t bitbuf_stride_words,
                                                         const unsigned long long *__restrict__ total_bits,
                                                         unsigned long long *__restrict__ lb_desc, uint32_t *__restrict__ ticket,
                                                         uint8_t *__restrict__ out, size_t out_stride, size_t out_capacity,
                                                         const unsigned long long *__restrict__ out_start, unsigned long long *__restrict__ out_next,
                                                         uint32_t *__restrict__ scan_size, uint32_t *__restrict__ status,
                                                         const uint32_t *__restrict__ mark, size_t mark_stride_words)
{
  __shared__ __align__(16) uint8_t stage[2 * STUFF_TILE_WORDS * 4 + 16];
  __shared__ unsigned ws[8];
  __shared__ unsigned long long s_base;
  __shared__ int s_tile, s_over;
  const int img = blockIdx.y;
  if (threadIdx.x == 0) { s_tile = (int)atomicAdd(&ticket[img], 1u); s_over = 0; }
  __syncthreads();
  const int tile = s_tile;
  unsigned long long *desc = lb_desc + (size_t)img * gridDim.x;
  const unsigned long long start = out_start[img];
  const unsigned long long bits = total_bits[img], nbytes = (bits + 7) >> 3;
  const unsigned long long tile0 = (unsigned long long)tile * STUFF_TILE_WORDS;
  if (tile0 * 4 >= nbytes && tile != 0) return;                      // past the stream: never a live tile's predecessor
  const bool last = tile0 * 4 + STUFF_TILE_WORDS * 4 >= nbytes;       // holds the last stream byte (or the stream is empty)
  if (status[img] & ~1u) {                                            // an earlier stage flagged this image: publish, store nothing
    if (threadIdx.x == 0) {
      lb_publish(desc + tile, tile == 0 ? LB_INC : LB_AGG);
      if (tile == 0) { scan_size[img] = 0; out_next[img] = start; }
    }
    return;
  }
  const unsigned padbits = (unsigned)(nbytes * 8 - bits);
  const unsigned long long w0 = tile0 + threadIdx.x * 4;
  int nb;
  const uint4 q = stuff_load(bitbuf + (size_t)img * bitbuf_stride_words, nbytes, padbits, w0, nb);
  const unsigned mk = marker_bits16(mark ? mark + (size_t)img * mark_stride_words : nullptr, w0);
  const unsigned ff = count_ff16(q, nb, mk);
  unsigned tot;
  const unsigned before = cta_excl_scan_256(ff, ws, tot);
  if (threadIdx.x < 32) {
    unsigned long long base = 0;
    if (tile > 0) { if (threadIdx.x == 0) lb_publish(desc + tile, LB_AGG | tot); base = lb_lookback(desc, tile); }
    if (threadIdx.x == 0) { lb_publish(desc + tile, LB_INC | (base + tot)); s_base = base; }
  }
  __syncthreads();
  const unsigned long long o0 = start + tile0 * 4 + s_base;          // output offset of the tile's first byte
  uint8_t *dst = out + (size_t)img * out_stride + o0;
  const int ph = (int)((uintptr_t)dst & 15);
  const int pos = threadIdx.x * 16 + (int)before;                    // this thread's first byte inside the tile's output
  if (nb) {
    if (o0 + pos + 32 > out_capacity) s_over = 1;
    const unsigned w[4] = {q.x, q.y, q.z, q.w};
    uint8_t *sp = stage + ph + pos;
#pragma unroll
    for (int j = 0; j < 16; j++) {
      if (j < nb) {
        const unsigned b = (w[j >> 2] >> (24 - 8 * (j & 3))) & 0xFF;
        *sp++ = (uint8_t)b;
        if (b == 0xFF && !((mk >> j) & 1u)) *sp++ = 0;
      }
    }
  }
  const unsigned long long tile_bytes = min(nbytes - tile0 * 4, (unsigned long long)STUFF_TILE_WORDS * 4);
  const int len = (int)(tile_bytes + tot), span = ph + len;
  __syncthreads();
  if (s_over) { if (threadIdx.x == 0) atomicOr(&status[img], 4u); }
  else {
    uint8_t *base = dst - ph;                                         // 16-byte aligned; bytes [ph, span) are the tile's
    for (int k = threadIdx.x; k * 16 < span; k += blockDim.x) {
      const int b0 = k * 16;
      if (b0 >= ph && b0 + 16 <= span) *reinterpret_cast<uint4 *>(base + b0) = *reinterpret_cast<const uint4 *>(stage + b0);
      else for (int i = max(b0, ph); i < min(b0 + 16, span); i++) base[i] = stage[i];
    }
  }
  if (last && threadIdx.x == 0) {
    const unsigned long long total = nbytes + s_base + tot;
    scan_size[img] = (uint32_t)total;
    out_next[img] = start + total;
  }
}
// =====================================================================
// progressive scans (jcphuff.c).  DC scans walk blocks in MCU order like
// the sequential coder.  AC scans are non-interleaved; their cross-block
// state (EOBRUN, and in refinement scans the buffered correction bits with
// the forced flush of jcphuff.c:998-1000) is resolved in three steps:
//   k_prog_flags : per block  brk (the block calls emit_eobrun before one of
//                  its own symbols), contrib (the block ends with EOBRUN++),
//                  tailBR (correction bits it appends to the pending run);
//   k_prog_runs  : one walker per breaker (and one for the scan start) follows
//                  the non-breaking blocks after it, applies the 0x7FFF /
//                  BE>937 forced flushes, and stores each sub-run's EOBRUN value
//                  at the sub-run's FIRST block;
//   walk_prog_ac : every block then emits, in stream order, its own symbols,
//                  the EOBRUN symbol it owns, and its tail correction bits.
// =====================================================================
#define AUX_BRK 1u
#define AUX_CONTRIB 2u

// Per block of an AC scan, three 64-bit position masks (bit i = zigzag position i, only positions of the band):
//   ev  : the coefficient is an event of the scan -- (|v| >> Al) != 0
//   one : refinement scans, (|v| >> Al) == 1 (newly nonzero: run symbol + sign bit)
//   bit : refinement scans, the bit the event sends -- sign for a 'one' (1 = positive, jcphuff.c:983), else the
//         correction bit (|v| >> Al) & 1
// kept in three planes [plane][img][block] so that the three symbol walks of the scan (statistics, bit counts, bit
// emission) visit only the events instead of all 63 positions.  Only the 16-byte pieces of the 128-byte block that
// the band touches are fetched -- a 1..8 scan moves one 32-byte sector per block.
__global__ void __launch_bounds__(256) k_prog_flags(Geom g, ScanDesc sd, uint32_t *__restrict__ aux, uint32_t *__restrict__ run_e,
                                                    unsigned long long *__restrict__ pm, int *__restrict__ tile_last, int *__restrict__ tile_first)
{
  __shared__ int smax[8], smin[8];
  int img = blockIdx.y;
  const int Al = sd.al_img ? sd.al_img[img] : sd.Al;     // scan search: this scan's Al is the image's best Al so far (jcmaster.c:477-488)
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  int bmax = -1, bmin = 0x7fffffff;
  if (t < sd.nblocks) {
    int sci, k; long long mcu;
    const int16_t *blk = block_ptr(g, sd, img, t, sci, mcu, k);
    const uint4 *b4 = reinterpret_cast<const uint4 *>(blk);
    unsigned evl = 0, evh = 0, onel = 0, oneh = 0, bitl = 0, bith = 0;
    const bool refine = sd.Ah != 0;
#pragma unroll
    for (int q = 0; q < 8; q++) {
      if (!(8 * q + 7 >= sd.Ss && 8 * q <= sd.Se)) continue;
      const uint4 a = b4[q];
      const unsigned w[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
      for (int j = 0; j < 8; j++) {
        const int i = 8 * q + j;
        const int v = (j & 1) ? (int)w[j >> 1] >> 16 : (int)(short)(w[j >> 1] & 0xFFFF);
        const int sft = abs(v) >> Al;
        const unsigned m = 1u << (i & 31);
        unsigned &ev = i < 32 ? evl : evh, &one = i < 32 ? onel : oneh, &bit = i < 32 ? bitl : bith;
        if (sft != 0) ev |= m;
        if (refine) {
          if (sft == 1) one |= m;
          if (sft == 1 ? v >= 0 : (sft & 1)) bit |= m;
        }
      }
    }
    const unsigned long long band = (sd.Se == 63 ? ~0ull : ((1ull << (sd.Se + 1)) - 1)) & ~((1ull << sd.Ss) - 1);
    const unsigned long long ev = (((unsigned long long)evh << 32) | evl) & band;
    const unsigned long long one = (((unsigned long long)oneh << 32) | onel) & ev;
    const unsigned long long bit = (((unsigned long long)bith << 32) | bitl) & ev;
    unsigned brk, contrib, tail = 0;
    if (!refine) {
      brk = ev != 0;
      contrib = !brk || (63 - __clzll((long long)ev)) != sd.Se;
    } else {
      brk = one != 0;
      const int lastone = brk ? 63 - __clzll((long long)one) : 0;
      tail = __popcll(ev & ~one & ~((2ull << lastone) - 1));         // correction bits after the last newly-nonzero coefficient
      contrib = lastone != sd.Se;
    }
    const size_t plane = (size_t)gridDim.y * sd.nblocks, at = (size_t)img * sd.nblocks + t;
    pm[at] = ev;
    if (refine) { pm[plane + at] = one; pm[2 * plane + at] = bit; }
    aux[at] = brk | (contrib << 1) | (tail << 2);
    run_e[at] = 0;
    if (brk || t == 0 || (sd.ri && t % sd.ri == 0)) bmax = bmin = (int)t;
  }
  for (int o = 16; o; o >>= 1) { bmax = max(bmax, __shfl_xor_sync(0xffffffffu, bmax, o)); bmin = min(bmin, __shfl_xor_sync(0xffffffffu, bmin, o)); }
  if ((threadIdx.x & 31) == 0) { smax[threadIdx.x >> 5] = bmax; smin[threadIdx.x >> 5] = bmin; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < 8; i++) { bmax = max(bmax, smax[i]); bmin = min(bmin, smin[i]); }
    tile_last[(size_t)img * gridDim.x + blockIdx.x] = bmax; tile_first[(size_t)img * gridDim.x + blockIdx.x] = bmin;
  }
}
// per image: tile_last -> running maximum over the tiles up to and including each tile; tile_first -> running
// minimum over the tiles from each tile to the end
__global__ void __launch_bounds__(256) k_prog_tile_scan(int ntiles, int *__restrict__ tile_last, int *__restrict__ tile_first)
{
  int *tl = tile_last + (size_t)blockIdx.x * ntiles, *tf = tile_first + (size_t)blockIdx.x * ntiles;
  __shared__ int carry, wsm[8];
  if (threadIdx.x == 0) carry = -1;
  __syncthreads();
  for (int base = 0; base < ntiles; base += 256) {
    int i = base + threadIdx.x, v = i < ntiles ? tl[i] : -1;
    for (int o = 1; o < 32; o <<= 1) { int y = __shfl_up_sync(0xffffffffu, v, o); if ((threadIdx.x & 31) >= o) v = max(v, y); }
    if ((threadIdx.x & 31) == 31) wsm[threadIdx.x >> 5] = v;
    __syncthreads();
    int pre = carry;
    for (int w = 0; w < (int)(threadIdx.x >> 5); w++) pre = max(pre, wsm[w]);
    v = max(v, pre);
    if (i < ntiles) tl[i] = v;
    __syncthreads();
    if (threadIdx.x == 255) carry = v;
    __syncthreads();
  }
  if (threadIdx.x == 0) carry = 0x7fffffff;
  __syncthreads();
  for (int base = 0; base < ntiles; base += 256) {             // from the last tile backwards
    int i = ntiles - 1 - (base + threadIdx.x), v = i >= 0 ? tf[i] : 0x7fffffff;
    for (int o = 1; o < 32; o <<= 1) { int y = __shfl_up_sync(0xffffffffu, v, o); if ((threadIdx.x & 31) >= o) v = min(v, y); }
    if ((threadIdx.x & 31) == 31) wsm[threadIdx.x >> 5] = v;
    __syncthreads();
    int pre = carry;
    for (int w = 0; w < (int)(threadIdx.x >> 5); w++) pre = min(pre, wsm[w]);
    v = min(v, pre);
    if (i >= 0) tf[i] = v;
    __syncthreads();
    if (threadIdx.x == 255) carry = v;
    __syncthreads();
  }
}
// EOBRUN values of a FIRST scan (Ah == 0: no correction bits, so a run is only cut every 0x7FFF blocks,
// jcphuff.c:727-729): every member of a run knows the run's start (last boundary at or before it) and end (next
// boundary after it); the first block of each sub-run of 0x7FFF members owns the sub-run's EOBRUN symbol.
__global__ void __launch_bounds__(256) k_prog_runs_first(ScanDesc sd, const uint32_t *__restrict__ aux, uint32_t *__restrict__ run_e,
                                                         const int *__restrict__ tile_last, const int *__restrict__ tile_first)
{
  __shared__ int sprev[8], snext[8];
  const int img = blockIdx.y, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t *a = aux + (size_t)img * sd.nblocks;
  unsigned f = 0; bool boundary = false;
  if (t < sd.nblocks) { f = a[t]; boundary = (f & AUX_BRK) || t == 0 || (sd.ri && t % sd.ri == 0); }
  // last boundary at or before t inside the tile / first boundary after t inside the tile
  int pv = boundary ? (int)t : -1;
  for (int o = 1; o < 32; o <<= 1) { int y = __shfl_up_sync(0xffffffffu, pv, o); if (lane >= o) pv = max(pv, y); }
  int nv = boundary ? (int)t : 0x7fffffff;
  for (int o = 1; o < 32; o <<= 1) { int y = __shfl_down_sync(0xffffffffu, nv, o); if (lane + o < 32) nv = min(nv, y); }
  int nstrict = __shfl_down_sync(0xffffffffu, nv, 1); if (lane == 31) nstrict = 0x7fffffff;
  if (lane == 31) sprev[wid] = pv;
  if (lane == 0) snext[wid] = nv;
  __syncthreads();
  for (int w = 0; w < wid; w++) pv = max(pv, sprev[w]);
  for (int w = wid + 1; w < 8; w++) nstrict = min(nstrict, snext[w]);
  if (t >= sd.nblocks) return;
  const int *tl = tile_last + (size_t)img * gridDim.x, *tf = tile_first + (size_t)img * gridDim.x;
  if (pv < 0) pv = tl[blockIdx.x - 1];                               // block 0 is a boundary, so tile 0 always has one
  if (nstrict == 0x7fffffff && blockIdx.x + 1 < gridDim.x) nstrict = tf[blockIdx.x + 1];
  const long long nb = nstrict == 0x7fffffff ? sd.nblocks : (long long)nstrict;
  const long long b = pv;
  const unsigned fb = (b == t) ? f : a[b];
  const bool b_brk = fb & AUX_BRK;
  const long long cb = b_brk ? ((fb & AUX_CONTRIB) ? 1 : 0) : 0;
  // members of the run: the boundary itself unless it is a breaker that does not end in an EOB, then every block up to nb
  const long long first_member = b_brk ? (cb ? b : b + 1) : b;
  if (t < first_member) return;
  const long long off = t - first_member, total = nb - first_member;
  if (off % 0x7FFF == 0) run_e[(size_t)img * sd.nblocks + t] = (uint32_t)min(0x7FFFLL, total - off);
}

__global__ void __launch_bounds__(256) k_prog_runs(ScanDesc sd, const uint32_t *__restrict__ aux, uint32_t *__restrict__ run_e)
{
  int img = blockIdx.y;
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= sd.nblocks) return;
  const uint32_t *a = aux + (size_t)img * sd.nblocks;
  uint32_t *re = run_e + (size_t)img * sd.nblocks;
  unsigned f = a[t];
  // a restart boundary flushes the pending run (emit_restart -> emit_eobrun, jcphuff.c:446), so a new run
  // starts at the first block of every restart segment (AC scans: one block per MCU)
  const long long seg = sd.ri;
  if (!(f & AUX_BRK) && t != 0 && !(seg && t % seg == 0)) return;
  unsigned E = 0, B = 0; long long first = -1, j;
  if (f & AUX_BRK) { if (f & AUX_CONTRIB) { E = 1; B = f >> 2; first = t; } j = t + 1; }
  else j = t;
  const long long j0 = j;
  for (; j < sd.nblocks; j++) {
    if (seg && j % seg == 0 && !(j == j0 && j == t)) break;
    unsigned fj = a[j];
    if (fj & AUX_BRK) break;
    if (E == 0) first = j;
    E += 1; B += fj >> 2;
    if (E == 0x7FFF || B > 937) { re[first] = E; E = 0; B = 0; }     // jcphuff.c:727-729, :998-1000
  }
  if (E > 0) re[first] = E;
}

// One block of a progressive scan, in stream order.  Sink: dc(nbits, bits),
// ac(symbol, nbits, bits), raw(bits, n).  AC scans walk the block's event masks (k_prog_flags): the zero runs are the
// gaps between consecutive events, and a first scan fetches only the coefficients it codes.
template <class Sink>
__device__ __forceinline__ void flush_corrections(Sink &sink, unsigned long long &br, int &nbr)
{
  if (nbr > 32) sink.raw((unsigned)(br >> 32), nbr - 32);
  if (nbr) sink.raw((unsigned)br, nbr > 32 ? 32 : nbr);
  br = 0; nbr = 0;
}
template <class Sink>
__device__ __forceinline__ void walk_prog_block(const int16_t *__restrict__ blk, const ScanDesc &sd, const int Al, int last_dc_shifted,
                                                unsigned aux, unsigned runE, unsigned long long ev, unsigned long long one,
                                                unsigned long long bit, Sink &sink)
{
  if (sd.Ss == 0) {
    int dc = (int)blk[0] >> Al;                       // arithmetic shift (jcphuff.c:497)
    if (sd.Ah == 0) {                                    // encode_mcu_DC_first :468-548
      int temp = dc - last_dc_shifted, temp2 = temp;
      if (temp < 0) { temp = -temp; temp2--; }
      sink.dc(nbits_of(temp), temp2);
    } else sink.raw((unsigned)dc & 1u, 1);               // encode_mcu_DC_refine :746-786
    return;
  }
  if (sd.Ah == 0) {                                      // encode_mcu_AC_first :648-737
    int prev = sd.Ss - 1;
    while (ev) {                                         // ev != 0 <=> the block breaks the pending EOB run
      const int i = __ffsll((long long)ev) - 1;
      ev &= ev - 1;
      int r = i - prev - 1; prev = i;
      int temp = blk[i], temp2 = temp >> 31;
      temp = (temp ^ temp2) - temp2; temp >>= Al;
      temp2 ^= temp;
      while (r > 15) { sink.ac(0xF0, 0, 0); r -= 16; }
      int nb = nbits_of(temp);
      sink.ac((r << 4) + nb, nb, temp2);
    }
    if (runE) { int nb = nbits_of((int)runE) - 1; sink.ac(nb << 4, nb, (int)runE); }   // emit_eobrun :409-431
    return;
  }
  // encode_mcu_AC_refine :817-1017
  unsigned long long br = 0; int nbr = 0;
  if (aux & AUX_BRK) {
    const int EOB = 63 - __clzll((long long)one);
    int prev = sd.Ss - 1, r = 0;
    while (ev) {
      const int i = __ffsll((long long)ev) - 1;
      ev &= ev - 1;
      r += i - prev - 1; prev = i;
      const unsigned b = (unsigned)(bit >> i) & 1u;
      while (r > 15 && i <= EOB) { sink.ac(0xF0, 0, 0); r -= 16; flush_corrections(sink, br, nbr); }
      if (!((one >> i) & 1)) { br = (br << 1) | b; nbr++; continue; }
      sink.ac((r << 4) + 1, 0, 0);
      sink.raw(b, 1);
      flush_corrections(sink, br, nbr);
      r = 0;
    }
  } else {
    nbr = __popcll(ev);
    while (ev) { const int i = __ffsll((long long)ev) - 1; ev &= ev - 1; br = (br << 1) | ((unsigned)(bit >> i) & 1u); }
  }
  // the EOBRUN symbol this block owns, then this block's tail correction bits
  if (runE) { int nb = nbits_of((int)runE) - 1; sink.ac(nb << 4, nb, (int)runE); }
  flush_corrections(sink, br, nbr);
}

__device__ __forceinline__ int prev_dc_shifted(const Geom &g, const ScanDesc &sd, const int Al, int img, long long t, int sci, long long mcu, int k)
{
  if (sd.Ss != 0 || sd.Ah != 0) return 0;
  long long tp;
  if (k > sd.k_first[sci]) tp = t - 1;
  else if (mcu > 0 && !(sd.ri && mcu % sd.ri == 0)) tp = t - sd.bim + sd.k_count[sci] - 1;   // jcphuff.c:455-457
  else return 0;
  int s2, k2; long long m2;
  const int16_t *p = block_ptr(g, sd, img, tp, s2, m2, k2);
  return (int)p[0] >> Al;
}

__device__ __forceinline__ void load_prog_aux(const ScanDesc &sd, const uint32_t *__restrict__ aux, const uint32_t *__restrict__ run_e,
                                              const unsigned long long *__restrict__ pm, int img, long long t, unsigned &a, unsigned &re,
                                              unsigned long long &ev, unsigned long long &one, unsigned long long &bit)
{
  const size_t plane = (size_t)gridDim.y * sd.nblocks, at = (size_t)img * sd.nblocks + t;
  a = aux[at]; re = run_e[at]; ev = pm[at];
  if (sd.Ah != 0) { one = pm[plane + at]; bit = pm[2 * plane + at]; }
}

struct HistSinkP {
  unsigned *dc_hist, *ac_hist; int bad; int maxbits;
  __device__ void dc(int nb, int) { if (nb > maxbits + 1) bad = 1; atomicAdd(&dc_hist[nb], 1u); }
  // a value's size against max_coef_bits (jcphuff.c:633); an EOBRUN symbol (low nibble 0) carries up to 14 run bits
  __device__ void ac(int sym, int nb, int) { if (nb > 14 || ((sym & 15) && nb > maxbits)) bad = 1; atomicAdd(&ac_hist[sym], 1u); }
  __device__ void raw(unsigned, int) {}
};
struct CountSinkP {
  const uint8_t *dsz, *asz; unsigned bits; int bad;
  __device__ void dc(int nb, int) { int s = dsz[nb]; if (!s) bad = 1; bits += s + nb; }
  __device__ void ac(int sym, int nb, int) { int s = asz[sym]; if (!s) bad = 1; bits += s + nb; }
  __device__ void raw(unsigned, int n) { bits += n; }
};
struct BitSinkP : BitSink {
  __device__ void raw(unsigned v, int n) { if (n == 32) { put(v >> 16, 16); put(v & 0xFFFFu, 16); } else put(v, n); }
};

__global__ void __launch_bounds__(256) k_gather_prog(Geom g, ScanDesc sd, const uint32_t *__restrict__ aux, const uint32_t *__restrict__ run_e,
                                                     const unsigned long long *__restrict__ pm, uint32_t *__restrict__ hist, uint32_t *__restrict__ status)
{
  __shared__ unsigned sh[GATHER_COPIES_SCAN][HIST_SLOTS * HIST_BINS];
  int img = blockIdx.y;
  const int Al = sd.al_img ? sd.al_img[img] : sd.Al;     // scan search: this scan's Al is the image's best Al so far (jcmaster.c:477-488)
  for (int i = threadIdx.x; i < GATHER_COPIES_SCAN * HIST_SLOTS * HIST_BINS; i += blockDim.x) (&sh[0][0])[i] = 0;
  __syncthreads();
#pragma unroll 1
  for (int tile = 0; tile < GATHER_TILES; tile++) {
    long long t = ((long long)blockIdx.x * GATHER_TILES + tile) * blockDim.x + threadIdx.x;
    if (t >= sd.nblocks) break;
    int sci, k; long long mcu;
    const int16_t *blk = block_ptr(g, sd, img, t, sci, mcu, k);
    int last = prev_dc_shifted(g, sd, Al, img, t, sci, mcu, k);
    const CompGeom &c = g.c[sd.ci[sci]];
    unsigned *mine = sh[threadIdx.x % GATHER_COPIES_SCAN];
    HistSinkP sink{mine + c.dc_tbl * HIST_BINS, mine + (4 + c.ac_tbl) * HIST_BINS, 0, g.max_coef_bits};
    unsigned a = 0, re = 0; unsigned long long ev = 0, one = 0, bit = 0;
    if (sd.Ss) load_prog_aux(sd, aux, run_e, pm, img, t, a, re, ev, one, bit);
    walk_prog_block(blk, sd, Al, last, a, re, ev, one, bit, sink);
    if (sink.bad) atomicOr(&status[img], 2u);
  }
  __syncthreads();
  uint32_t *gh = hist + (size_t)img * HIST_SLOTS * HIST_BINS;
  for (int i = threadIdx.x; i < HIST_SLOTS * HIST_BINS; i += blockDim.x) {
    unsigned v = 0;
#pragma unroll
    for (int cp = 0; cp < GATHER_COPIES_SCAN; cp++) v += sh[cp][i];
    if (v) atomicAdd(&gh[i], v);
  }
}

__global__ void __launch_bounds__(256) k_block_bits_prog(Geom g, ScanDesc sd, const DevHuff *__restrict__ tabs, size_t stride,
                                                         const uint32_t *__restrict__ aux, const uint32_t *__restrict__ run_e,
                                                         const unsigned long long *__restrict__ pm, uint32_t *__restrict__ blk_bits, uint32_t *__restrict__ tile_bits, uint32_t *__restrict__ status)
{
  __shared__ ScanTables st;
  __shared__ unsigned ws[8];
  int img = blockIdx.y;
  const int Al = sd.al_img ? sd.al_img[img] : sd.Al;     // scan search: this scan's Al is the image's best Al so far (jcmaster.c:477-488)
  if (!(sd.Ss == 0 && sd.Ah != 0)) load_scan_tables(st, tabs, stride, img, g, sd, false);
  __syncthreads();
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  unsigned bits = 0;
  if (t < sd.nblocks) {
    int sci, k; long long mcu;
    const int16_t *blk = block_ptr(g, sd, img, t, sci, mcu, k);
    int last = prev_dc_shifted(g, sd, Al, img, t, sci, mcu, k);
    const CompGeom &c = g.c[sd.ci[sci]];
    CountSinkP sink{st.size[c.dc_tbl], st.size[4 + c.ac_tbl], 0u, 0};
    unsigned a = 0, re = 0; unsigned long long ev = 0, one = 0, bit = 0;
    if (sd.Ss) load_prog_aux(sd, aux, run_e, pm, img, t, a, re, ev, one, bit);
    walk_prog_block(blk, sd, Al, last, a, re, ev, one, bit, sink);
    if (sink.bad) atomicOr(&status[img], 2u);
    bits = sink.bits;
  }
  unsigned tot;
  const unsigned pre = cta_excl_scan_256(bits, ws, tot);
  if (t < sd.nblocks) blk_bits[(size_t)img * sd.nblocks + t] = pre;
  if (threadIdx.x == 0) tile_bits[(size_t)img * gridDim.x + blockIdx.x] = tot;
}

__global__ void __launch_bounds__(256) k_encode_prog(Geom g, ScanDesc sd, const DevHuff *__restrict__ tabs, size_t stride,
                                                     const uint32_t *__restrict__ aux, const uint32_t *__restrict__ run_e,
                                                     const unsigned long long *__restrict__ pm,
                                                     const uint32_t *__restrict__ blk_bits, const uint32_t *__restrict__ tile_bits /* per-tile totals: not read here */,
                                                     const unsigned long long *__restrict__ tile_base,
                                                     const uint32_t *__restrict__ seg_corr, long long seg_stride,
                                                     uint32_t *__restrict__ bitbuf, size_t bitbuf_stride_words,
                                                     uint32_t *__restrict__ mark, size_t mark_stride_words, const uint32_t *__restrict__ status)
{
  __shared__ ScanTables st;
  int img = blockIdx.y;
  const int Al = sd.al_img ? sd.al_img[img] : sd.Al;     // scan search: this scan's Al is the image's best Al so far (jcmaster.c:477-488)
  if (!(sd.Ss == 0 && sd.Ah != 0)) load_scan_tables(st, tabs, stride, img, g, sd, true);
  __syncthreads();
  if (status[img] & ~1u) return;
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned long long tb = tile_base[(size_t)img * gridDim.x + blockIdx.x];
  uint32_t *gbuf = bitbuf + (size_t)img * bitbuf_stride_words;
  if (t < sd.nblocks) {
    unsigned long long off = tb + blk_bits[(size_t)img * sd.nblocks + t];
    if (sd.ri) off += seg_corr[(size_t)img * seg_stride + t / ((long long)sd.ri * sd.bim)];
    int sci, k; long long mcu;
    const int16_t *blk = block_ptr(g, sd, img, t, sci, mcu, k);
    int last = prev_dc_shifted(g, sd, Al, img, t, sci, mcu, k);
    const CompGeom &c = g.c[sd.ci[sci]];
    BitSinkP sink;
    sink.buf = gbuf; sink.widx = off >> 5; sink.acc = 0; sink.nacc = (int)(off & 31);
    sink.dco = st.code[c.dc_tbl]; sink.aco = st.code[4 + c.ac_tbl]; sink.dsz = st.size[c.dc_tbl]; sink.asz = st.size[4 + c.ac_tbl];
    unsigned a = 0, re = 0; unsigned long long ev = 0, one = 0, bit = 0;
    if (sd.Ss) load_prog_aux(sd, aux, run_e, pm, img, t, a, re, ev, one, bit);
    walk_prog_block(blk, sd, Al, last, a, re, ev, one, bit, sink);
    if (sd.ri) emit_restart_marker(sink, sd, t, mark + (size_t)img * mark_stride_words);
    sink.finish();
  }
}


// =====================================================================
// scan search (optimize_scans), successive-approximation part of select_scans
// (jcmaster.c:773-962): pick, per image, the point transform Al that minimises
// the size of {band scans at Al} + {refinement scans below Al}, with the
// reference's early stop at the first non-improvement.  A scan's size is what
// the reference buffers for it: DHT + SOS + entropy-coded bytes.
//   first      : index of the first Al-search scan of the group
//   per_al     : scans per Al step (luma 3: refine, low band, high band; chroma 6)
//   nband      : band scans per step (luma 2, chroma 4); nrefine = per_al - nband
// =====================================================================
__device__ __forceinline__ unsigned scan_total_bytes(const ScanDesc &sd, const Geom &g, const DevHuff *t /* this image's 8 slots for the scan */, unsigned entropy_bytes)
{
  unsigned dht = 0; unsigned seen = 0;
  for (int i = 0; i < sd.ncomps; i++) {
    const CompGeom &c = g.c[sd.ci[i]];
    if (sd.Ss == 0 && sd.Ah == 0 && !((seen >> c.dc_tbl) & 1u)) { seen |= 1u << c.dc_tbl; dht += 17 + t[c.dc_tbl].nsym16; }
    if (sd.Se != 0 && !((seen >> (4 + c.ac_tbl)) & 1u)) { seen |= 1u << (4 + c.ac_tbl); dht += 17 + t[4 + c.ac_tbl].nsym16; }
  }
  if (dht) dht += 4;                                   // one DHT marker holds all of the scan's tables (emit_multi_dht, jcmarker.c:293-401)
  return dht + (sd.dri ? 6 : 0) + (2 + 2 + 1 + 2 * sd.ncomps + 3) + entropy_bytes;
}
__global__ void k_select_al(Geom g, AlSearch as, const DevHuff *__restrict__ tabs_scan, const uint32_t *__restrict__ scan_size, int n, int *__restrict__ best_al)
{
  const int img = blockIdx.x * blockDim.x + threadIdx.x;
  if (img >= n) return;
  const DevHuff *timg = tabs_scan + (size_t)img * as.nscans_total * HIST_SLOTS;
  auto size_of = [&](int si) -> unsigned long long {
    return scan_total_bytes(as.sd[si - as.first], g, timg + (size_t)si * HIST_SLOTS, scan_size[(size_t)si * n + img]);
  };
  const int nref = as.per_al - as.nband;
  unsigned long long best = 0; int best_Al = 0;
  for (int Al = 0; Al <= as.al_max; Al++) {
    // band scans at this Al: the group starts with the nband scans at Al = 0, then per step {refinements, bands at Al+1}
    const int band0 = Al == 0 ? as.first : as.first + as.nband + (Al - 1) * as.per_al + nref;
    unsigned long long cost = 0;
    for (int b = 0; b < as.nband; b++) cost += size_of(band0 + b);
    for (int i = 0; i < Al; i++) for (int r = 0; r < nref; r++) cost += size_of(as.first + as.nband + i * as.per_al + r);
    if (Al == 0 || cost < best) { best = cost; best_Al = Al; }
    else break;                                          // jcmaster.c:800-803 / :861-864
  }
  best_al[img] = best_Al;
}
void launch_select_al(const Geom &g, const AlSearch &as, const DevHuff *tabs_scan, const uint32_t *scan_size, int n, int *best_al, cudaStream_t s)
{
  k_select_al<<<(n + 63) / 64, 64, 0, s>>>(g, as, tabs_scan, scan_size, n, best_al);
  LAUNCHED();
}

void launch_prog_prepare(const Geom &g, const ScanDesc &sd, uint32_t *aux, uint32_t *run_e, unsigned long long *pm, int *tile_last, int *tile_first, int n, cudaStream_t s)
{
  if (sd.Ss == 0) return;
  dim3 grid((unsigned)((sd.nblocks + 255) / 256), n);
  k_prog_flags<<<grid, 256, 0, s>>>(g, sd, aux, run_e, pm, tile_last, tile_first); LAUNCHED();
  if (sd.Ah == 0) {
    k_prog_tile_scan<<<n, 256, 0, s>>>((int)grid.x, tile_last, tile_first); LAUNCHED();
    k_prog_runs_first<<<grid, 256, 0, s>>>(sd, aux, run_e, tile_last, tile_first); LAUNCHED();
  } else { k_prog_runs<<<grid, 256, 0, s>>>(sd, aux, run_e); LAUNCHED(); }
}
void launch_gather_prog(const Geom &g, const ScanDesc &sd, const uint32_t *aux, const uint32_t *run_e, const unsigned long long *pm, uint32_t *hist, uint32_t *status, int n, cudaStream_t s)
{
  dim3 grid((unsigned)((sd.nblocks + 256 * GATHER_TILES - 1) / (256 * GATHER_TILES)), n);
  k_gather_prog<<<grid, 256, 0, s>>>(g, sd, aux, run_e, pm, hist, status); LAUNCHED();
}

void launch_block_bits(const Geom &g, const ScanDesc &sd, const DcRec *nz_rec, const uint8_t *sym, const int16_t *dcq, const RecLayout &rl, const DevHuff *tabs, size_t stride, int progressive,
                       uint32_t *blk_bits, uint32_t *tile_bits, const uint32_t *blk_aux, const uint32_t *run_e, const unsigned long long *pm, uint32_t *status, int n, cudaStream_t s)
{
  dim3 grid((unsigned)((sd.nblocks + 255) / 256), n);
  if (progressive) k_block_bits_prog<<<grid, 256, 0, s>>>(g, sd, tabs, stride, blk_aux, run_e, pm, blk_bits, tile_bits, status);
  else k_block_bits_seq<<<grid, 256, 0, s>>>(g, sd, nz_rec, sym, dcq, rl, tabs, stride, blk_bits, tile_bits, status);
  LAUNCHED();
}
void launch_scan_layout(const ScanDesc &sd, const uint32_t *blk_bits, const uint32_t *tile_bits, unsigned long long *tile_base,
                        uint32_t *seg_corr, long long seg_stride, unsigned long long *total_bits, size_t capacity_bits,
                        uint32_t *status, int n, cudaStream_t s)
{
  const int ntiles = (int)((sd.nblocks + 255) / 256);
  k_scan_layout<<<n, 256, 0, s>>>(sd, blk_bits, tile_bits, ntiles, tile_base, seg_corr, seg_stride, total_bits, capacity_bits, status);
  LAUNCHED();
}
// the packers OR their bits into a zeroed word stream: only the words the scan will occupy (total_bits is known since
// k_scan_layout) are cleared, not the whole worst-case buffer
__global__ void __launch_bounds__(256) k_zero_stream(uint32_t *__restrict__ bitbuf, size_t stride_words, const unsigned long long *__restrict__ total_bits)
{
  const int img = blockIdx.y;
  const unsigned long long need = min((unsigned long long)stride_words, ((total_bits[img] + 31) >> 5) + 8) + 3 >> 2;      // 16-byte pieces
  uint4 *dst = reinterpret_cast<uint4 *>(bitbuf + (size_t)img * stride_words);
  const unsigned long long stride4 = stride_words >> 2;
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const unsigned long long q = ((unsigned long long)blockIdx.x * 4 + j) * 256 + threadIdx.x;
    if (q < need && q < stride4) dst[q] = make_uint4(0, 0, 0, 0);
  }
}
void launch_zero_stream(uint32_t *bitbuf, size_t stride_words, const unsigned long long *total_bits, int n, cudaStream_t s)
{
  dim3 grid((unsigned)((stride_words / 4 + 1023) / 1024), n);
  k_zero_stream<<<grid, 256, 0, s>>>(bitbuf, stride_words, total_bits); LAUNCHED();
}
void launch_encode(const Geom &g, const ScanDesc &sd, const DcRec *nz_rec, const uint8_t *sym, const int16_t *dcq, const RecLayout &rl, const DevHuff *tabs, size_t stride, int progressive,
                   const uint32_t *blk_bits, const uint32_t *tile_bits, const unsigned long long *tile_base, const uint32_t *seg_corr, long long seg_stride,
                   const uint32_t *blk_aux, const uint32_t *run_e, const unsigned long long *pm,
                   uint32_t *bitbuf, size_t bitbuf_stride_words, uint32_t *mark, size_t mark_stride_words, const uint32_t *status, int n, cudaStream_t s)
{
  dim3 grid((unsigned)((sd.nblocks + 255) / 256), n);
  if (progressive) k_encode_prog<<<grid, 256, 0, s>>>(g, sd, tabs, stride, blk_aux, run_e, pm, blk_bits, tile_bits, tile_base, seg_corr, seg_stride, bitbuf, bitbuf_stride_words, mark, mark_stride_words, status);
  else k_encode_seq<<<grid, 256, 0, s>>>(g, sd, nz_rec, sym, dcq, rl, tabs, stride, blk_bits, tile_bits, tile_base, seg_corr, seg_stride, bitbuf, bitbuf_stride_words, mark, mark_stride_words, status);
  LAUNCHED();
}
// =====================================================================
// lossless (SOF3) coding: prediction + point transform (jclossls.c:43-250, jcdiffct.c:156-232) and the lossless
// Huffman coder (jclhuff.c:316-530).  One MCU = one sample of each scan component (all components are 1x1 in lossless
// mode, jcmaster.c:1079-1081); MCU t of a scan is the pixel (t % W, t / W).
// =====================================================================
// sample `k` of the pixel at px, unmasked as the null-type conversions leave it (jccolor.c:604-715 apply no
// RANGE_LIMIT): 8-bit JSAMPLE, 12-bit J12SAMPLE (signed short), 16-bit J16SAMPLE (unsigned short).  The C-ABI takes
// pitches, strides and pointers with no alignment, so a 16-bit sample is assembled from its two bytes (little endian).
template <int PREC>
__device__ __forceinline__ int ll_sample(const uint8_t *__restrict__ px, int k)
{
  if (PREC == 8) return (int)__ldg(px + k);
  const unsigned short v = (unsigned short)(__ldg(px + 2 * k) | (unsigned)__ldg(px + 2 * k + 1) << 8);
  return PREC == 12 ? (int)(short)v : (int)v;
}
// category (0..16) of a difference taken mod 2^16, and the value bits that follow it (jclhuff.c:356-391): the magnitude
// is masked with 0x7FFF; -32768 mod 2^16 is category 16 with no value bits (the temp == 0 case at :361-369)
__device__ __forceinline__ int ll_category(unsigned d16, unsigned &vbits)
{
  if (d16 & 0x8000u) {
    const unsigned m = (0u - d16) & 0x7FFFu;
    vbits = ~m;
    return m ? 32 - __clz(m) : 16;
  }
  vbits = d16;
  return d16 ? 32 - __clz(d16) : 0;
}

// The differences of one scan: diff[(img * ncomps + i) * W*H + t] for scan component i, and the categories counted into
// hist[img][dc_tbl][0..16] (encode_mcus_gather, jclhuff.c:460-524) through a per-CTA histogram.
// Row y restarts the prediction (first-row predictors) when y is a multiple of the rows per restart interval: reset_predictor
// fires when restart_rows_to_go reaches 0, and the first-row differencer keeps itself for the next row exactly then
// (jclossls.c:73-79, :111-114, :200-232); without restarts only row 0 is a first row.
template <int PREC>
__global__ void __launch_bounds__(256) k_lossless_diff(Geom g, ScanDesc sd, const uint8_t *__restrict__ src,
                                                       uint16_t *__restrict__ diff, uint32_t *__restrict__ hist)
{
  __shared__ unsigned sh[4][17];
  for (int i = threadIdx.x; i < 4 * 17; i += blockDim.x) sh[i / 17][i % 17] = 0;
  __syncthreads();
  const int img = blockIdx.y;
  const long long npix = (long long)g.W * g.H;
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < npix) {
    const int y = (int)(t / g.W), x = (int)(t - (long long)y * g.W);
    const int rows_per_restart = sd.ri ? sd.ri / g.W : 0;
    const bool first_row = rows_per_restart ? (y % rows_per_restart) == 0 : y == 0;
    constexpr int SB = PREC == 8 ? 1 : 2;
    const size_t pxb = (size_t)g.in_comps * SB;
    const uint8_t *row = src + (size_t)img * g.image_stride + (size_t)y * g.row_pitch;
    const uint8_t *up = row - g.row_pitch;
    const int Al = sd.Al;
    for (int i = 0; i < sd.ncomps; i++) {
      const int c = sd.ci[i];
      const int k = g.px_first + (g.px_swap ? 2 - c : c);          // the RGB-family orders (jccolor.c:253-291); k = c otherwise
      const int samp = ll_sample<PREC>(row + x * pxb, k) >> Al;      // RIGHT_SHIFT by Pt (jclossls.c:255-262)
      int pred;
      if (first_row) pred = x == 0 ? 1 << (PREC - Al - 1) : ll_sample<PREC>(row + (x - 1) * pxb, k) >> Al;
      else {
        const int Rb = ll_sample<PREC>(up + x * pxb, k) >> Al;
        if (x == 0) pred = Rb;
        else {
          const int Ra = ll_sample<PREC>(row + (x - 1) * pxb, k) >> Al, Rc = ll_sample<PREC>(up + (x - 1) * pxb, k) >> Al;
          switch (sd.Ss) {                                          // PREDICTOR1..7 (jlossls.h:37-43)
          case 1: pred = Ra; break;
          case 2: pred = Rb; break;
          case 3: pred = Rc; break;
          case 4: pred = Ra + Rb - Rc; break;
          case 5: pred = Ra + ((Rb - Rc) >> 1); break;
          case 6: pred = Rb + ((Ra - Rc) >> 1); break;
          default: pred = (Ra + Rb) >> 1; break;
          }
        }
      }
      const unsigned d16 = (unsigned)(samp - pred) & 0xFFFFu;
      diff[((size_t)img * sd.ncomps + i) * npix + t] = (uint16_t)d16;
      unsigned vb;
      atomicAdd(&sh[g.c[c].dc_tbl][ll_category(d16, vb)], 1u);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 4 * 17; i += blockDim.x) {
    const unsigned v = sh[i / 17][i % 17];
    if (v) atomicAdd(&hist[((size_t)img * HIST_SLOTS + i / 17) * HIST_BINS + i % 17], v);
  }
}

// bits of every MCU (category codes + value bits), exclusive prefix inside the 256-MCU tile and the tile sums, in the
// layout k_scan_layout reads
__global__ void __launch_bounds__(256) k_lossless_bits(Geom g, ScanDesc sd, const uint16_t *__restrict__ diff,
                                                       const DevHuff *__restrict__ tabs, size_t stride,
                                                       uint32_t *__restrict__ blk_bits, uint32_t *__restrict__ tile_bits, uint32_t *__restrict__ status)
{
  __shared__ uint8_t size[4][17];
  __shared__ unsigned ws[9];
  const int img = blockIdx.y;
  const DevHuff *t8 = reinterpret_cast<const DevHuff *>(reinterpret_cast<const char *>(tabs) + (size_t)img * stride);
  for (int i = threadIdx.x; i < 4 * 17; i += blockDim.x) size[i / 17][i % 17] = t8[i / 17].size[i % 17];
  __syncthreads();
  const long long npix = (long long)g.W * g.H;
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  unsigned bits = 0; int bad = 0;
  if (t < npix) {
    for (int i = 0; i < sd.ncomps; i++) {
      unsigned vb;
      const int nb = ll_category(diff[((size_t)img * sd.ncomps + i) * npix + t], vb);
      const int sz = size[g.c[sd.ci[i]].dc_tbl][nb];
      if (!sz) bad = 1;
      bits += sz + (nb == 16 ? 0 : nb);
    }
  }
  if (bad) atomicOr(&status[img], 2u);
  unsigned tot;
  const unsigned pre = cta_excl_scan_256(bits, ws, tot);
  if (t < npix) blk_bits[(size_t)img * npix + t] = pre;
  if (threadIdx.x == 0) tile_bits[(size_t)img * gridDim.x + blockIdx.x] = tot;
}

// pack every MCU at its offset; restart markers as k_encode_seq writes them (emit_restart, jclhuff.c:286-309)
__global__ void __launch_bounds__(256) k_lossless_encode(Geom g, ScanDesc sd, const uint16_t *__restrict__ diff,
                                                         const DevHuff *__restrict__ tabs, size_t stride,
                                                         const uint32_t *__restrict__ blk_bits, const unsigned long long *__restrict__ tile_base,
                                                         const uint32_t *__restrict__ seg_corr, long long seg_stride,
                                                         uint32_t *__restrict__ bitbuf, size_t bitbuf_stride_words,
                                                         uint32_t *__restrict__ mark, size_t mark_stride_words, const uint32_t *__restrict__ status)
{
  __shared__ uint32_t cs[4][17];             // code | size << 16
  const int img = blockIdx.y;
  const DevHuff *t8 = reinterpret_cast<const DevHuff *>(reinterpret_cast<const char *>(tabs) + (size_t)img * stride);
  for (int i = threadIdx.x; i < 4 * 17; i += blockDim.x) cs[i / 17][i % 17] = (uint32_t)t8[i / 17].code[i % 17] | (uint32_t)t8[i / 17].size[i % 17] << 16;
  __syncthreads();
  if (status[img] & ~1u) return;            // an earlier stage flagged this image (overflow / missing code)
  const long long npix = (long long)g.W * g.H;
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= npix) return;
  unsigned long long off = tile_base[(size_t)img * gridDim.x + blockIdx.x] + blk_bits[(size_t)img * npix + t];
  if (sd.ri) off += seg_corr[(size_t)img * seg_stride + t / sd.ri];
  BitSink sink;
  sink.buf = bitbuf + (size_t)img * bitbuf_stride_words; sink.widx = off >> 5; sink.acc = 0; sink.nacc = (int)(off & 31);
  for (int i = 0; i < sd.ncomps; i++) {
    unsigned vb;
    const int nb = ll_category(diff[((size_t)img * sd.ncomps + i) * npix + t], vb);
    const uint32_t e = cs[g.c[sd.ci[i]].dc_tbl][nb];
    const int vn = nb == 16 ? 0 : nb;
    sink.put(((e & 0xFFFFu) << vn) | (vb & ((1u << vn) - 1u)), (int)(e >> 16) + vn);
  }
  if (sd.ri) emit_restart_marker(sink, sd, t, mark + (size_t)img * mark_stride_words);
  sink.finish();
}

void launch_lossless_diff(const Geom &g, const ScanDesc &sd, int precision, const uint8_t *src, uint16_t *diff, uint32_t *hist, int n, cudaStream_t s)
{
  dim3 grid((unsigned)(((long long)g.W * g.H + 255) / 256), n);
  if (precision == 8) k_lossless_diff<8><<<grid, 256, 0, s>>>(g, sd, src, diff, hist);
  else if (precision == 12) k_lossless_diff<12><<<grid, 256, 0, s>>>(g, sd, src, diff, hist);
  else k_lossless_diff<16><<<grid, 256, 0, s>>>(g, sd, src, diff, hist);
  LAUNCHED();
}
void launch_lossless_bits(const Geom &g, const ScanDesc &sd, const uint16_t *diff, const DevHuff *tabs, size_t stride,
                          uint32_t *blk_bits, uint32_t *tile_bits, uint32_t *status, int n, cudaStream_t s)
{
  dim3 grid((unsigned)(((long long)g.W * g.H + 255) / 256), n);
  k_lossless_bits<<<grid, 256, 0, s>>>(g, sd, diff, tabs, stride, blk_bits, tile_bits, status);
  LAUNCHED();
}
void launch_lossless_encode(const Geom &g, const ScanDesc &sd, const uint16_t *diff, const DevHuff *tabs, size_t stride,
                            const uint32_t *blk_bits, const unsigned long long *tile_base, const uint32_t *seg_corr, long long seg_stride,
                            uint32_t *bitbuf, size_t bitbuf_stride_words, uint32_t *mark, size_t mark_stride_words, const uint32_t *status, int n, cudaStream_t s)
{
  dim3 grid((unsigned)(((long long)g.W * g.H + 255) / 256), n);
  k_lossless_encode<<<grid, 256, 0, s>>>(g, sd, diff, tabs, stride, blk_bits, tile_base, seg_corr, seg_stride, bitbuf, bitbuf_stride_words, mark, mark_stride_words, status);
  LAUNCHED();
}

size_t stuff_tiles(size_t bitbuf_stride_words) { return (bitbuf_stride_words + STUFF_TILE_WORDS - 1) / STUFF_TILE_WORDS; }
size_t stuff_lookback_bytes(size_t bitbuf_stride_words, int n) { return (size_t)n * 8 + (size_t)n * stuff_tiles(bitbuf_stride_words) * 8; }
void launch_stuff(const uint32_t *bitbuf, size_t bitbuf_stride_words, const unsigned long long *total_bits, void *lookback,
                  uint8_t *out, size_t out_stride, size_t out_capacity, const unsigned long long *out_start, unsigned long long *out_next,
                  uint32_t *scan_size, uint32_t *status, const uint32_t *mark, size_t mark_stride_words, int n, cudaStream_t s)
{
  dim3 grid((unsigned)stuff_tiles(bitbuf_stride_words), n);
  unsigned long long *desc = static_cast<unsigned long long *>(lookback);
  uint32_t *ticket = reinterpret_cast<uint32_t *>(desc + (size_t)n * grid.x);
  k_stuff<<<grid, STUFF_THREADS, 0, s>>>(bitbuf, bitbuf_stride_words, total_bits, desc, ticket, out, out_stride, out_capacity, out_start, out_next, scan_size, status, mark, mark_stride_words);
  LAUNCHED();
}

}  // namespace b200

namespace b200 {

// ================================================================ sequential Huffman decode (jpeg_read_coefficients)
// Speculative decode with self-synchronisation over DEC_SUB_BITS-bit subsequences of every restart segment (decode.cuh).
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
  if (col >= o.wib[c] || row >= o.hib[c]) return nullptr;          // a dummy block of an interleaved scan
  return o.plane[c] + (((long long)sc.img * o.hib[c] + row) * o.wib[c] + col) * 64;
}

// one thread per subsequence: decode again from the synchronised start and write the AC coefficients of every block
// that starts inside the subsequence (finishing the last one past its end) into the planes (zeroed before), the DC
// differences into dcd; the segment's last subsequence checks that the segment holds all its MCUs
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
  long long blk = (long long)(dec_prefix(pre, tsum, j) - seg_base);
  if (j == g.sub0 + g.nsub - 1 && blk + (long long)r.count < need) atomicOr(&status[sc.img], 1u);
  const uint32_t b = min((uint32_t)(j - g.sub0 + 1) * DEC_SUB_BITS, g.nbits);
  uint32_t pos = r.in_pos, st = r.in_st;
  bool skip = (st & 127) != 0 && st != DEC_DEAD;         // the block in progress belongs to the predecessor
  int16_t *dst = nullptr;
  while (st != DEC_DEAD && blk < need) {
    if ((st & 127) == 0) {                                // a block starts here
      if (pos >= b) break;
      dst = dec_block(*o, sc, g.mcu0 + blk / sc.nb, (int)(st >> 7));
    }
    int zz, val; bool done;
    st = dec_step(w, g.nbits, pos, st, sc, tabs, zz, val, done);
    if (st == DEC_DEAD) break;
    if (!skip) {
      if (zz == 0) dcd[g.blk0 + blk] = val;
      else if (zz > 0 && dst) dst[c_zz[zz]] = (int16_t)val;
    }
    if (done) { blk++; skip = false; }
  }
}

// one warp per (segment, scan component): DC values = running sum of the differences over the component's blocks in
// scan order, dummy blocks included, reset at the segment start (decode_mcu: int accumulation, JCOEF store)
__global__ void __launch_bounds__(128) k_dec_dc(const DecSeg *__restrict__ segs, int nsegs, const DecScan *__restrict__ scans,
                                                const int *__restrict__ dcd, const DecOut *__restrict__ o)
{
  const long long gw = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (gw >= (long long)nsegs * 4) return;
  const DecSeg g = segs[gw >> 2];
  const int k = (int)(gw & 3);
  const DecScan &sc = scans[g.scan];
  if (k >= sc.ncomp) return;
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
    if (e < total) { int16_t *dst = dec_block(*o, sc, g.mcu0 + m, slot); if (dst) dst[0] = (int16_t)s; }
    carry = __shfl_sync(0xffffffffu, s, 31);
  }
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

// jpeg_idct_islow (jidctint.c:171-419, 8-bit: CONST_BITS 13, PASS1_BITS 2) with the dequantization of jddctmgr.c:
// 134-146 (ISLOW_MULT_TYPE is a short: the table entries are taken as int16).  Eight lanes per block: each loads one
// 16-byte row of the JBLOCK, transforms one column into the int workspace (pass 1), then one row into eight samples
// (pass 2) stored as one 8-byte word.  The reference's shortcuts for all-zero columns and rows give what the general
// butterfly gives, so there is no branch.  Pass 1 keeps the reference's 64-bit intermediates (JLONG): a file may carry
// 16-bit coefficients under a 16-bit table; pass 2 needs bits 18..27 of its sums only, which 32-bit arithmetic keeps.
// coef: [nblocks][64] natural order ([n][hib][wib] blocks); quant: image i's table at quant + i * qstride;
// out: [n][hib * 8][wib * 8] samples.
__global__ void __launch_bounds__(IDCT_BLOCKS * 8) k_idct_islow(const int16_t *__restrict__ coef, const uint16_t *__restrict__ quant, int qstride,
                                                                uint8_t *__restrict__ out, int wib, int hib, long long nblocks)
{
  __shared__ int4 s_coef[IDCT_BLOCKS * 8];
  __shared__ int s_ws[IDCT_BLOCKS * IDCT_WS];
  const int lb = threadIdx.x >> 3, lane = threadIdx.x & 7;
  const long long blk = (long long)blockIdx.x * IDCT_BLOCKS + lb;
  const bool valid = blk < nblocks;
  const long long per = (long long)wib * hib;
  const long long img = valid ? blk / per : 0;
  s_coef[threadIdx.x] = valid ? reinterpret_cast<const int4 *>(coef)[blk * 8 + lane] : make_int4(0, 0, 0, 0);
  __syncwarp();
  // pass 1: column `lane`
  {
    const int16_t *c = reinterpret_cast<const int16_t *>(s_coef + lb * 8) + lane;
    const uint16_t *q = quant + img * qstride + lane;
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
      const long long rem = blk - img * per;
      const int by = (int)(rem / wib), bx = (int)(rem - (long long)by * wib);
      uint8_t *dst = out + ((img * hib + by) * 8 + lane) * ((long long)wib * 8) + bx * 8;
      *reinterpret_cast<uint2 *>(dst) = make_uint2(o0 | o1 << 8 | o2 << 16 | o3 << 24, o4 | o5 << 8 | o6 << 16 | o7 << 24);
    }
  }
}

void launch_idct_islow(const int16_t *coef, const uint16_t *quant, int qstride, uint8_t *out, int wib, int hib, int n, cudaStream_t s)
{
  const long long nblocks = (long long)n * wib * hib;
  k_idct_islow<<<(unsigned)((nblocks + IDCT_BLOCKS - 1) / IDCT_BLOCKS), IDCT_BLOCKS * 8, 0, s>>>(coef, quant, qstride, out, wib, hib, nblocks); LAUNCHED();
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
// out: [n][hib * N][wib * N] samples.
template <int N>
__global__ void __launch_bounds__(IDCT_BLOCKS * 8) k_idct_red(const int16_t *__restrict__ coef, const uint16_t *__restrict__ quant, int qstride,
                                                              uint8_t *__restrict__ out, int wib, int hib, long long nblocks)
{
  const long long per = (long long)wib * hib;
  if (N == 1) {
    const long long blk = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (blk >= nblocks) return;
    const long long img = blk / per, rem = blk - img * per;
    const int by = (int)(rem / wib), bx = (int)(rem - (long long)by * wib);
    const int dq = (int)__ldg(coef + blk * 64) * (int)__ldg(quant + img * qstride);
    out[(img * hib + by) * (long long)wib + bx] = (uint8_t)idct_range_limit((int)(((long long)dq + 4) >> 3));
    return;
  }
  __shared__ int4 s_coef[IDCT_BLOCKS * 8];
  __shared__ int s_ws[IDCT_BLOCKS * IDCT_WS];
  const int lb = threadIdx.x >> 3, lane = threadIdx.x & 7;
  const long long blk = (long long)blockIdx.x * IDCT_BLOCKS + lb;
  const bool valid = blk < nblocks;
  const long long img = valid ? blk / per : 0;
  s_coef[threadIdx.x] = valid ? reinterpret_cast<const int4 *>(coef)[blk * 8 + lane] : make_int4(0, 0, 0, 0);
  __syncwarp();
  const bool col_used = N == 4 ? lane != 4 : (lane & 1) || lane == 0;
  if (col_used) {                                         // pass 1: column `lane` -> ws rows 0 .. N-1
    const int16_t *c = reinterpret_cast<const int16_t *>(s_coef + lb * 8) + lane;
    const uint16_t *q = quant + img * qstride + lane;
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
  if (valid && lane < N) {                                // pass 2: row `lane`
    const int *w = s_ws + lb * IDCT_WS + lane * 9;
    const long long rem = blk - img * per;
    const int by = (int)(rem / wib), bx = (int)(rem - (long long)by * wib);
    uint8_t *dst = out + ((img * hib + by) * N + lane) * ((long long)wib * N) + bx * N;
    if (N == 4) {
      const long long t0 = (long long)w[0] * 16384, t2 = (long long)w[2] * 15137 + (long long)w[6] * -6270;
      const long long tmp10 = t0 + t2, tmp12 = t0 - t2;
      const long long z1 = w[7], z2 = w[5], z3 = w[3], z4 = w[1];
      const long long o0 = z1 * -1730 + z2 * 11893 + z3 * -17799 + z4 * 8697;
      const long long o2 = z1 * -4176 + z2 * -4926 + z3 * 7373 + z4 * 20995;
      const long long rnd = 1LL << 18;
      const unsigned s0 = idct_range_limit((int)((tmp10 + o2 + rnd) >> 19)), s3 = idct_range_limit((int)((tmp10 - o2 + rnd) >> 19));
      const unsigned s1 = idct_range_limit((int)((tmp12 + o0 + rnd) >> 19)), s2 = idct_range_limit((int)((tmp12 - o0 + rnd) >> 19));
      *reinterpret_cast<uint32_t *>(dst) = s0 | s1 << 8 | s2 << 16 | s3 << 24;
    } else {
      const long long tmp10 = (long long)w[0] * 32768;
      const long long o0 = (long long)w[7] * -5906 + (long long)w[5] * 6967 + (long long)w[3] * -10426 + (long long)w[1] * 29692;
      const long long rnd = 1LL << 19;
      const unsigned s0 = idct_range_limit((int)((tmp10 + o0 + rnd) >> 20)), s1 = idct_range_limit((int)((tmp10 - o0 + rnd) >> 20));
      *reinterpret_cast<uint16_t *>(dst) = (uint16_t)(s0 | s1 << 8);
    }
  }
}

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
__global__ void __launch_bounds__(IDCT_BLOCKS * 8) k_idct_ifast(const int16_t *__restrict__ coef, const int *__restrict__ mtab, int qstride,
                                                                uint8_t *__restrict__ out, int wib, int hib, long long nblocks)
{
  __shared__ int4 s_coef[IDCT_BLOCKS * 8];
  __shared__ int s_ws[IDCT_BLOCKS * IDCT_WS];
  const int lb = threadIdx.x >> 3, lane = threadIdx.x & 7;
  const long long blk = (long long)blockIdx.x * IDCT_BLOCKS + lb;
  const bool valid = blk < nblocks;
  const long long per = (long long)wib * hib;
  const long long img = valid ? blk / per : 0;
  s_coef[threadIdx.x] = valid ? reinterpret_cast<const int4 *>(coef)[blk * 8 + lane] : make_int4(0, 0, 0, 0);
  __syncwarp();
  {
    const int16_t *c = reinterpret_cast<const int16_t *>(s_coef + lb * 8) + lane;
    const int *q = mtab + img * qstride + lane;
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
      const long long rem = blk - img * per;
      const int by = (int)(rem / wib), bx = (int)(rem - (long long)by * wib);
      uint8_t *dst = out + ((img * hib + by) * 8 + lane) * ((long long)wib * 8) + bx * 8;
      *reinterpret_cast<uint2 *>(dst) = make_uint2(s[0] | s[1] << 8 | s[2] << 16 | s[3] << 24, s[4] | s[5] << 8 | s[6] << 16 | s[7] << 24);
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
__global__ void __launch_bounds__(IDCT_BLOCKS * 8) k_idct_float(const int16_t *__restrict__ coef, const float *__restrict__ mtab, int qstride,
                                                                uint8_t *__restrict__ out, int wib, int hib, long long nblocks)
{
  __shared__ int4 s_coef[IDCT_BLOCKS * 8];
  __shared__ float s_ws[IDCT_BLOCKS * IDCT_WS];
  const int lb = threadIdx.x >> 3, lane = threadIdx.x & 7;
  const long long blk = (long long)blockIdx.x * IDCT_BLOCKS + lb;
  const bool valid = blk < nblocks;
  const long long per = (long long)wib * hib;
  const long long img = valid ? blk / per : 0;
  s_coef[threadIdx.x] = valid ? reinterpret_cast<const int4 *>(coef)[blk * 8 + lane] : make_int4(0, 0, 0, 0);
  __syncwarp();
  {
    const int16_t *c = reinterpret_cast<const int16_t *>(s_coef + lb * 8) + lane;
    const float *q = mtab + img * qstride + lane;
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
      const long long rem = blk - img * per;
      const int by = (int)(rem / wib), bx = (int)(rem - (long long)by * wib);
      uint8_t *dst = out + ((img * hib + by) * 8 + lane) * ((long long)wib * 8) + bx * 8;
      *reinterpret_cast<uint2 *>(dst) = make_uint2(s[0] | s[1] << 8 | s[2] << 16 | s[3] << 24, s[4] | s[5] << 8 | s[6] << 16 | s[7] << 24);
    }
  }
}

void launch_idct_opts(int size, int method, const int16_t *coef, const void *tab, int qstride, uint8_t *out, int wib, int hib, int n, cudaStream_t s)
{
  const long long nblocks = (long long)n * wib * hib;
  const unsigned grid8 = (unsigned)((nblocks + IDCT_BLOCKS - 1) / IDCT_BLOCKS);
  const uint16_t *q = static_cast<const uint16_t *>(tab);
  if (size == 1) { k_idct_red<1><<<(unsigned)((nblocks + 255) / 256), 256, 0, s>>>(coef, q, qstride, out, wib, hib, nblocks); LAUNCHED(); }
  else if (size == 2) { k_idct_red<2><<<grid8, IDCT_BLOCKS * 8, 0, s>>>(coef, q, qstride, out, wib, hib, nblocks); LAUNCHED(); }
  else if (size == 4) { k_idct_red<4><<<grid8, IDCT_BLOCKS * 8, 0, s>>>(coef, q, qstride, out, wib, hib, nblocks); LAUNCHED(); }
  else if (method == 1) { k_idct_ifast<<<grid8, IDCT_BLOCKS * 8, 0, s>>>(coef, static_cast<const int *>(tab), qstride, out, wib, hib, nblocks); LAUNCHED(); }
  else if (method == 2) { k_idct_float<<<grid8, IDCT_BLOCKS * 8, 0, s>>>(coef, static_cast<const float *>(tab), qstride, out, wib, hib, nblocks); LAUNCHED(); }
  else launch_idct_islow(coef, q, qstride, out, wib, hib, n, s);
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
__global__ void __launch_bounds__(256) k_upsample_opts(UpsOpt o, uint8_t *__restrict__ pix, long long row_pitch, long long image_stride, int W, int H)
{
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y, img = blockIdx.z;
  if (x >= W || y >= H) return;
  int v[3] = {0, 0, 0};
#pragma unroll
  for (int c = 0; c < 3; c++)
    if (c < o.nin) v[c] = up_one(o.plane[c] + img * o.stride[c], o.pitch[c], o.dw[c], o.dh[c], o.hr[c], o.vr[c], o.fancy[c] != 0, x, y);
  uint8_t *d = pix + img * image_stride + (long long)y * row_pitch + (long long)x * o.ps;
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

void launch_upsample_opts(const UpsOpt &o, uint8_t *pix, size_t row_pitch, size_t image_stride, int W, int H, int n, cudaStream_t s)
{
  const dim3 cta(64, 4), grid((unsigned)((W + 63) / 64), (unsigned)((H + 3) / 4), (unsigned)n);
  k_upsample_opts<<<grid, cta, 0, s>>>(o, pix, (long long)row_pitch, (long long)image_stride, W, H); LAUNCHED();
}

}  // namespace b200
