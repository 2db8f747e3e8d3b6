// decompress.cu -- host side of the decompressor: the entropy decode of a batch of JPEG files into coefficient planes,
// the IDCT / upsampling / colour conversion to pixels or YUV planes, and the decompress, recompress, transcode and
// decode C-ABI entry points of include/b200jpeg.h over them.
#include "encoder.h"
#include "decode_kernels.cuh"
#include <climits>
#include <cstring>
#include <array>
#include <string>
#include <vector>

namespace b200 {

static uint32_t *dec_words_alloc(void *ctx, size_t words)
{
  b200jpeg_encoder *e = static_cast<b200jpeg_encoder *>(ctx);
  return e->h_dec_words.reserve(words * 4) ? nullptr : e->h_dec_words.as<uint32_t>();
}

static const char *const kDecStages[8] = {"dec_h2d", "dec_sync", "dec_fix", "dec_scan", "dec_write", "dec_dc", "dec_dc_refine", "dec_ac_refine"};

// the decode stages of the last decode, appended to the stage times (the refinements after a progressive decode)
static void add_decode_stage_times(b200jpeg_encoder *e)
{
  for (int k = 0; k < (e->dec_prog ? 8 : 6); k++) {
    float ms = 0.f; cudaEventElapsedTime(&ms, e->dec_ev[k], e->dec_ev[k + 1]);
    e->stage_names.push_back(kDecStages[k]); e->stage_ms.push_back(ms); e->stage_calls.push_back(1);
  }
}

// the decode stage times of the last decode, added to e->dec_ms
static void sum_decode_stage_times(b200jpeg_encoder *e)
{
  for (int k = 0; k < (e->dec_prog ? 8 : 6); k++) { float ms = 0.f; cudaEventElapsedTime(&ms, e->dec_ev[k], e->dec_ev[k + 1]); e->dec_ms[k < 6 ? k : k + 2] += ms; }
}

// Entropy decode of n files into e->d_dec_planes (jpeg_read_coefficients for the batch): the first scans through the
// speculative decode, then every DC refinement, then the AC refinement levels in order.
// first: the batch index of files[0], for the messages; mixed: the files may differ in geometry (DecBatch::mixed).
static int decode_files(b200jpeg_encoder *e, const uint8_t *const *files, const size_t *sizes, int n, int first = 0, bool mixed = false)
{
  if (!e || !files || !sizes || n <= 0) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  CU(cudaSetDevice(e->device));
  DecBatch &b = e->dec;
  b.progressive = e->progressive_decode;
  b.mixed = mixed;
  int rc = build_decode_batch(files, sizes, n, b, dec_words_alloc, e, first);
  if (rc) return rc;
  e->dec_prog = false;
  for (int i = 0; i < n; i++) e->dec_prog |= b.info[i].sof == 0xC2;
  const size_t nseg_all = b.segs.size() + b.dcr_segs.size() + b.acr_segs.size();
  size_t total = 0;
  for (int c = 0; c < 4; c++) { e->dec_plane_off[c] = total; total += ((size_t)b.plane_blocks[c] * 128 + 255) & ~(size_t)255; }
  const long long ntiles = (b.nsub + 1023) / 1024;
  if ((rc = e->d_dec_words.reserve(b.nwords * 4 + 16)) || (rc = e->d_dec_segs.reserve(nseg_all * sizeof(DecSeg))) ||
      (rc = e->d_dec_scans.reserve(b.scans.size() * sizeof(DecScan))) || (rc = e->d_dec_tabs.reserve(b.tabs.size() * sizeof(DecTable))) ||
      (rc = e->d_dec_out.reserve(sizeof(DecOut))) || (rc = e->d_dec_rec.reserve((size_t)b.nsub * sizeof(DecRec))) ||
      (rc = e->d_dec_pre.reserve((size_t)b.nsub * 4)) || (rc = e->d_dec_tsum.reserve((size_t)ntiles * 8)) ||
      (rc = e->d_dec_dcd.reserve((size_t)b.nblocks * 4 + 4)) || (rc = e->d_dec_planes.reserve(total)) ||
      (rc = e->d_dec_stat.reserve((size_t)n * 4 + 24)) || (rc = e->h_dec_stat.reserve((size_t)n * 4 + 24)))
    return rc;
  for (cudaEvent_t &ev : e->dec_ev) if (!ev) CU(cudaEventCreate(&ev));
  DecOut o; memset(&o, 0, sizeof o);
  for (int c = 0; c < 4; c++) if (b.plane_blocks[c]) o.plane[c] = reinterpret_cast<int16_t *>(e->d_dec_planes.as<uint8_t>() + e->dec_plane_off[c]);
  cudaStream_t s = e->stream;
  uint8_t *stat = e->d_dec_stat.as<uint8_t>();          // [n] status words, max rounds (int), resynchronised subsequences (u64)
  const size_t rounds_off = ((size_t)n * 4 + 7) & ~(size_t)7, stat_bytes = rounds_off + 16;
  CU(cudaEventRecord(e->dec_ev[0], s));
  CU(cudaMemcpyAsync(e->d_dec_words.p, e->h_dec_words.p, b.nwords * 4, cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(e->d_dec_segs.p, b.segs.data(), b.segs.size() * sizeof(DecSeg), cudaMemcpyHostToDevice, s));
  DecSeg *d_dcr = e->d_dec_segs.as<DecSeg>() + b.segs.size(), *d_acr = d_dcr + b.dcr_segs.size();
  if (!b.dcr_segs.empty()) CU(cudaMemcpyAsync(d_dcr, b.dcr_segs.data(), b.dcr_segs.size() * sizeof(DecSeg), cudaMemcpyHostToDevice, s));
  if (!b.acr_segs.empty()) CU(cudaMemcpyAsync(d_acr, b.acr_segs.data(), b.acr_segs.size() * sizeof(DecSeg), cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(e->d_dec_scans.p, b.scans.data(), b.scans.size() * sizeof(DecScan), cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(e->d_dec_tabs.p, b.tabs.data(), b.tabs.size() * sizeof(DecTable), cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(e->d_dec_out.p, &o, sizeof o, cudaMemcpyHostToDevice, s));
  CU(cudaMemsetAsync(e->d_dec_planes.p, 0, total, s));
  CU(cudaMemsetAsync(stat, 0, stat_bytes, s));
  launch_decode(e->d_dec_words.as<uint32_t>(), e->d_dec_segs.as<DecSeg>(), (int)b.segs.size(), e->d_dec_scans.as<DecScan>(), e->d_dec_tabs.as<DecTable>(), b.nsub,
                e->d_dec_rec.as<DecRec>(), e->d_dec_pre.as<uint32_t>(), e->d_dec_tsum.as<unsigned long long>(), e->d_dec_dcd.as<int>(), e->d_dec_out.as<DecOut>(),
                reinterpret_cast<uint32_t *>(stat), reinterpret_cast<int *>(stat + rounds_off), reinterpret_cast<unsigned long long *>(stat + rounds_off + 8),
                e->dec_ev + 1, s);
  if (e->dec_prog)
    launch_decode_refine(e->d_dec_words.as<uint32_t>(), d_dcr, (int)b.dcr_segs.size(), b.dcr_blocks, d_acr, b.acr_level.data(), (int)b.acr_level.size() - 1,
                         e->d_dec_scans.as<DecScan>(), e->d_dec_tabs.as<DecTable>(), e->d_dec_out.as<DecOut>(), reinterpret_cast<uint32_t *>(stat), e->dec_ev + 7, s);
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(e->h_dec_stat.p, stat, stat_bytes, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  const uint8_t *hs = e->h_dec_stat.as<uint8_t>();
  e->dec_rounds = *reinterpret_cast<const int *>(hs + rounds_off);
  e->dec_redone = (long long)*reinterpret_cast<const unsigned long long *>(hs + rounds_off + 8);
  for (int i = 0; i < n; i++) {
    const uint32_t st = reinterpret_cast<const uint32_t *>(hs)[i];
    if (st & 1) { set_error("image %d: corrupt entropy-coded data (an invalid Huffman code, or too few bits for a segment's MCUs)", first + i); return B200JPEG_ERR_BAD_SOURCE; }
    if (st & 2) { set_error("image %d: corrupt entropy-coded data (a coefficient past the end of its scan's spectral band)", first + i); return B200JPEG_ERR_BAD_SOURCE; }
    if (st & 4) { set_error("image %d: corrupt entropy-coded data (an AC refinement symbol whose size is not 1)", first + i); return B200JPEG_ERR_BAD_SOURCE; }
  }
  return B200JPEG_OK;
}

// jpegtran from file bytes (b200jpeg_transcode_batch, and with a transform b200jpeg_transcode_batch_transform)
static int transcode_files(b200jpeg_encoder *e, const b200jpeg_params *p, const b200jpeg_transform_info *t, const uint8_t *const *files, const size_t *sizes, int n_images)
{
  if (!e || !p) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  e->dec.want_markers = false;
  int rc = decode_files(e, files, sizes, n_images);
  if (rc) return rc;
  const DecBatch &b = e->dec;
  const DecGeom &g0 = b.geom[0];
  // -grayscale keeps the first component of a 3-component source; every other destination has the source's components
  const bool comps_ok = p->num_components == g0.nc || (t && t->force_grayscale && p->num_components == 1);
  if (!comps_ok) { set_error("the parameter block has %d components, the sources %d", p->num_components, g0.nc); return B200JPEG_ERR_PARAM; }
  if (t) {
    for (int c = 0; c < p->num_components; c++)
      if (t->src_wib[c] != g0.wib[c] || t->src_hib[c] != g0.hib[c]) { set_error("the sources' component %d has %dx%d blocks, the transform description %dx%d", c, g0.wib[c], g0.hib[c], t->src_wib[c], t->src_hib[c]); return B200JPEG_ERR_PARAM; }
  }
  // each image's quantization tables: what its components latched, in the slots p assigns them; in the source's
  // orientation (p's are transposed back), encode_coefs_xform transposes them with the blocks
  std::vector<uint16_t> qt((size_t)n_images * B200JPEG_NUM_QUANT_TBLS * 64);
  for (int i = 0; i < n_images; i++) {
    uint16_t *q = qt.data() + (size_t)i * B200JPEG_NUM_QUANT_TBLS * 64;
    memcpy(q, p->quant_tbl, sizeof p->quant_tbl);
    if (t && t->transposed) transpose_qsets(q, 1);
    for (int c = 0; c < p->num_components; c++) {
      const int slot = p->comp_info[c].quant_tbl_no;
      if (slot < 0 || slot >= B200JPEG_NUM_QUANT_TBLS || !b.info[i].comp_quant_present[c]) { set_error("image %d: Quantization table 0x%02x was not defined", i, slot); return B200JPEG_ERR_PARAM; }
      memcpy(q + slot * 64, b.info[i].comp_quant[c], 128);
    }
  }
  int16_t *planes[4]; size_t pitch[4], stride[4];
  for (int c = 0; c < 4; c++) {
    planes[c] = c < g0.nc ? reinterpret_cast<int16_t *>(e->d_dec_planes.as<uint8_t>() + e->dec_plane_off[c]) : nullptr;
    pitch[c] = c < g0.nc ? (size_t)g0.wib[c] : 0; stride[c] = c < g0.nc ? (size_t)g0.wib[c] * g0.hib[c] : 0;
  }
  rc = t ? encode_coefs_xform(e, p, t, planes, 1, pitch, stride, qt.data(), n_images)
         : b200jpeg_encode_batch_coefs_qtables(e, p, planes, 1, pitch, stride, qt.data(), n_images);
  if (rc) return rc;
  add_decode_stage_times(e);
  return B200JPEG_OK;
}

// what every decode to samples needs of a source beyond its layout: each component's table defined and, for a
// progressive file, a valid progression the reference would not block-smooth
static int check_tables_progression(const b200jpeg_source_info &s, int i)
{
  for (int c = 0; c < s.num_components; c++)
    if (!s.comp_quant_present[c]) { set_error("image %d: Quantization table 0x%02x was not defined", i, s.quant_tbl_no[c]); return B200JPEG_ERR_BAD_SOURCE; }
  if (s.sof == 0xC2) {
    int cb[4][64];
    if (int rc = check_progression(s, cb)) { std::string m = b200jpeg_last_error(); set_error("image %d: %s", i, m.c_str()); return rc; }
    if (smoothing_applies(s, cb)) {
      set_error("image %d: incomplete progression: the reference decompressor applies block smoothing to it (do_block_smoothing), which is not on the device path", i);
      return B200JPEG_ERR_UNSUPPORTED;
    }
  }
  return B200JPEG_OK;
}

// A source b200jpeg_decompress_batch takes: sequential (or, with progressive decode on, progressive without the block
// smoothing a default decompress object would apply), 8-bit, gray or three components with component 0 at the
// largest factors (1 or 2 each way) over 1x1 chroma, or, when every rung of the call sets cmyk, four components whose
// every sampling factor is 1 or 2 (a factor of 3 or 4 keeps the 4-component refusal); everything else is refused,
// never approximated.
static int check_decompress_source(const b200jpeg_source_info &s, int i, bool progressive, bool cmyk)
{
  bool four_ok = cmyk && s.num_components == 4;
  for (int c = 0; four_ok && c < 4; c++) four_ok = s.h_samp_factor[c] <= 2 && s.v_samp_factor[c] <= 2;
  const char *why = nullptr;
  if (s.sof == 0xC2 && !progressive) why = "progressive (SOF2) source: only sequential files are decoded to pixels";
  else if (s.data_precision != 8) why = "12-bit source: only 8-bit files are decoded to pixels";
  else if (s.num_components != 1 && s.num_components != 3 && !four_ok) why = "4-component (CMYK / YCCK) source: only gray and 3-component files are decoded to pixels";
  else if (s.num_components == 3 && (s.h_samp_factor[0] > 2 || s.v_samp_factor[0] > 2 || s.h_samp_factor[1] != 1 || s.v_samp_factor[1] != 1 ||
                                     s.h_samp_factor[2] != 1 || s.v_samp_factor[2] != 1))
    why = "sampling layout other than 4:4:4, 4:2:2, 4:4:0 or 4:2:0 (the reference's int_upsample and 2:1 non-fancy cases are not on the device)";
  if (why) { set_error("image %d: %s", i, why); return B200JPEG_ERR_UNSUPPORTED; }
  return check_tables_progression(s, i);
}

// the multiplier tables of jddctmgr.c start_pass for the ifast and float IDCTs, from one quantization table
static const int kAanScales[64] = {
  16384, 22725, 21407, 19266, 16384, 12873,  8867,  4520, 22725, 31521, 29692, 26722, 22725, 17855, 12299,  6270,
  21407, 29692, 27969, 25172, 21407, 16819, 11585,  5906, 19266, 26722, 25172, 22654, 19266, 15137, 10426,  5315,
  16384, 22725, 21407, 19266, 16384, 12873,  8867,  4520, 12873, 17855, 16819, 15137, 12873, 10114,  6967,  3552,
   8867, 12299, 11585, 10426,  8867,  6967,  4799,  2446,  4520,  6270,  5906,  5315,  4520,  3552,  2446,  1247};
static const double kAanScaleFactor[8] = {1.0, 1.387039845, 1.306562965, 1.175875602, 1.0, 0.785694958, 0.541196100, 0.275899379};
static void method_table(int method, const uint16_t *q, uint32_t *out)
{
  for (int i = 0; i < 64; i++) {
    if (method == B200JPEG_DCT_IFAST) {
      const int v = (int)(((long long)q[i] * kAanScales[i] + 2048) >> 12);                 // DESCALE(.., 14 - IFAST_SCALE_BITS)
      memcpy(&out[i], &v, 4);
    } else {
      const float f = (float)((double)q[i] * kAanScaleFactor[i >> 3] * kAanScaleFactor[i & 7]);
      memcpy(&out[i], &f, 4);
    }
  }
}

// the sample planes of one chunk's pixel stage for `plan`: per needed component nk images of hib x wib blocks of
// ssize x ssize samples; off[c]: where component c's plane starts.  Returns the bytes of all of them.
static size_t sample_plane_layout(const DecGeom &b, const DecPlan &plan, int nk, size_t off[4])
{
  size_t total = 0;
  for (int c = 0; c < 4; c++) off[c] = 0;
  for (int c = 0; c < b.nc; c++) {
    if (!plan.needed[c]) continue;
    off[c] = total; total += ((size_t)nk * b.hib[c] * b.wib[c] * plan.ssize[c] * plan.ssize[c] + 255) & ~(size_t)255;
  }
  return total;
}

// the device buffers one chunk's pixel stage for `plan` uses: sample planes, dequantization tables and, for the ifast
// and float IDCTs at full size, multiplier tables.  A chunk's pixel stages are enqueued back to back, so every plan is
// reserved for before the first is enqueued: no buffer is reallocated under a queued kernel.
static int reserve_pixel_stage(b200jpeg_encoder *e, const DecPlan &plan, int nk)
{
  const DecGeom &b = e->dec.geom[0];
  size_t off[4];
  bool need_mt = false;
  for (int c = 0; c < b.nc; c++) need_mt |= plan.needed[c] && plan.ssize[c] == 8 && plan.method != B200JPEG_DCT_ISLOW;
  int rc;
  if ((rc = e->d_dec_samples.reserve(sample_plane_layout(b, plan, nk, off))) || (rc = e->d_dec_quant.reserve((size_t)nk * b.nc * 128)) ||
      (need_mt && (rc = e->d_dec_mtab.reserve((size_t)nk * b.nc * 256)))) return rc;
  return B200JPEG_OK;
}

// the tables each image of the decoded chunk latched, [nk][qs][64] (qs: the most components of an image; slots past
// an image's components are zero), into e->d_dec_quant (qt: host staging)
static int upload_chunk_quant(b200jpeg_encoder *e, int nk, int qs, std::vector<uint16_t> &qt)
{
  const DecBatch &b = e->dec;
  qt.assign((size_t)nk * qs * 64, 0);
  for (int i = 0; i < nk; i++)
    for (int c = 0; c < b.geom[i].nc; c++) memcpy(&qt[((size_t)i * qs + c) * 64], b.info[i].comp_quant[c], 128);
  CU(cudaMemcpyAsync(e->d_dec_quant.p, qt.data(), qt.size() * 2, cudaMemcpyHostToDevice, e->stream));
  return B200JPEG_OK;
}

// the default plan's IDCT and upsampling / colour conversion of one decoded chunk: jpeg_idct_islow per component into
// planes of wib * 8 samples a row, then the fancy upsampling and default colour conversion into the pixels
static int idct_upsample_default(b200jpeg_encoder *e, int nk, uint8_t *pix, size_t row_pitch, size_t image_stride, const cudaEvent_t *ev)
{
  const DecGeom &b = e->dec.geom[0];
  const int nc = b.nc, W = b.W, H = b.H;
  const int hx = nc == 3 ? b.h[0] : 1, vx = nc == 3 ? b.v[0] : 1;
  cudaStream_t s = e->stream;
  size_t off[4];
  sample_plane_layout(b, DecPlan(), nk, off);
  CU(cudaEventRecord(ev[0], s));
  const uint8_t *planes[4] = {nullptr, nullptr, nullptr, nullptr}; int pitch[4] = {0, 0, 0, 0}; long long stride[4] = {0, 0, 0, 0};
  for (int c = 0; c < nc; c++) {
    uint8_t *dst = e->d_dec_samples.as<uint8_t>() + off[c];
    launch_idct_islow(reinterpret_cast<const int16_t *>(e->d_dec_planes.as<uint8_t>() + e->dec_plane_off[c]), e->d_dec_quant.as<uint16_t>() + c * 64, nc * 64,
                      dst, b.wib[c], b.hib[c], nk, s);
    planes[c] = dst; pitch[c] = b.wib[c] * 8; stride[c] = (long long)b.hib[c] * 8 * pitch[c];
  }
  CU(cudaEventRecord(ev[1], s));
  const int dw = div_up(W, hx), dh = div_up(H, vx);                    // downsampled_width / _height of the chroma (jdmaster.c)
  if (launch_upsample_color(hx, vx, nc, planes, pitch, stride, dw, dh, nc == 3 && e->dec.info[0].jpeg_color_space != B200JPEG_CS_RGB,
                            pix, row_pitch, image_stride, W, H, nk, s)) { set_error("no upsampling kernel for %dx%d sampling of %d components", hx, vx, nc); return B200JPEG_ERR_UNSUPPORTED; }
  CU(cudaEventRecord(ev[2], s));
  CU(cudaGetLastError());
  return B200JPEG_OK;
}

// component c of plan p in an upsampling descriptor: its sample plane (pitch bytes a row, images stride apart) and
// the plan's size, replication and filter for it
static void ups_component(UpsOpt4 &u, const DecPlan &p, int c, const uint8_t *plane, int pitch, long long stride)
{
  u.plane[c] = plane; u.pitch[c] = pitch; u.stride[c] = stride;
  u.dw[c] = p.dw[c]; u.dh[c] = p.dh[c]; u.hr[c] = p.hr[c]; u.vr[c] = p.vr[c]; u.fancy[c] = p.fancy[c];
}

static void ups_conversion(UpsOpt4 &u, const DecPlan &p)
{
  u.nin = p.nin; u.conv = p.conv; u.ps = p.ps;
  for (int k = 0; k < 4; k++) u.off[k] = p.off[k];
}

// the first three components of a descriptor, for the 1- and 3-component kernels (k_upsample_opts<3>, _ragged<3>)
static UpsOpt ups_narrow(const UpsOpt4 &a)
{
  UpsOpt o;
  memset(&o, 0, sizeof o);
  for (int c = 0; c < 3; c++) {
    o.plane[c] = a.plane[c]; o.pitch[c] = a.pitch[c]; o.stride[c] = a.stride[c];
    o.dw[c] = a.dw[c]; o.dh[c] = a.dh[c]; o.hr[c] = a.hr[c]; o.vr[c] = a.vr[c]; o.fancy[c] = a.fancy[c];
  }
  o.nin = a.nin; o.conv = a.conv; o.ps = a.ps;
  for (int k = 0; k < 4; k++) o.off[k] = a.off[k];
  return o;
}

// the IDCT and upsampling / colour conversion stages of one decoded chunk for a non-default plan: each needed
// component through the IDCT of its DCT_scaled_size into a plane of wib * size samples a row, then k_upsample_opts
// into the pixels.  qt: the chunk's tables as upload_chunk_quant staged them; mt: host staging for the multipliers.
static int idct_upsample_opts(b200jpeg_encoder *e, const DecPlan &plan, int nk, uint8_t *pix, size_t row_pitch, size_t image_stride,
                              const std::vector<uint16_t> &qt, std::vector<uint32_t> &mt, const cudaEvent_t *ev)
{
  const DecGeom &b = e->dec.geom[0];
  const int nc = b.nc;
  cudaStream_t s = e->stream;
  size_t off[4];
  sample_plane_layout(b, plan, nk, off);
  bool need_mt = false;
  for (int c = 0; c < nc; c++) need_mt |= plan.needed[c] && plan.ssize[c] == 8 && plan.method != B200JPEG_DCT_ISLOW;
  if (need_mt) {
    mt.resize((size_t)nk * nc * 64);
    for (size_t t = 0; t < (size_t)nk * nc; t++) method_table(plan.method, &qt[t * 64], &mt[t * 64]);
    CU(cudaMemcpyAsync(e->d_dec_mtab.p, mt.data(), mt.size() * 4, cudaMemcpyHostToDevice, s));
  }
  CU(cudaEventRecord(ev[0], s));
  UpsOpt4 u;
  memset(&u, 0, sizeof u);
  for (int c = 0; c < nc; c++) {
    if (!plan.needed[c]) continue;
    const int sz = plan.ssize[c];
    uint8_t *dst = e->d_dec_samples.as<uint8_t>() + off[c];
    const bool by_method = sz == 8 && plan.method != B200JPEG_DCT_ISLOW;
    const void *tab = by_method ? static_cast<const void *>(e->d_dec_mtab.as<uint32_t>() + c * 64) : static_cast<const void *>(e->d_dec_quant.as<uint16_t>() + c * 64);
    launch_idct_opts(sz, plan.method, reinterpret_cast<const int16_t *>(e->d_dec_planes.as<uint8_t>() + e->dec_plane_off[c]), tab, nc * 64, dst, b.wib[c], b.hib[c], nk, s);
    ups_component(u, plan, c, dst, b.wib[c] * sz, (long long)b.hib[c] * sz * b.wib[c] * sz);
  }
  CU(cudaEventRecord(ev[1], s));
  ups_conversion(u, plan);
  if (plan.nin == 4) launch_upsample_opts(u, pix, row_pitch, image_stride, plan.out_w, plan.out_h, nk, s);
  else launch_upsample_opts(ups_narrow(u), pix, row_pitch, image_stride, plan.out_w, plan.out_h, nk, s);
  CU(cudaEventRecord(ev[2], s));
  CU(cudaGetLastError());
  return B200JPEG_OK;
}

// Pixels for one DecPlan from the decoded chunk (e->dec, e->d_dec_planes, its tables in e->d_dec_quant) into (pix,
// row_pitch, image_stride): the default plan through launch_idct_islow and launch_upsample_color, every other plan
// through idct_upsample_opts.  A 4-component plan takes idct_upsample_opts whatever is_default says: the default
// route's k_upsample_color has no 4-component instance.  It only enqueues on e->stream, with events ev[0..2] around
// the IDCT and around the upsampling / colour conversion; the caller reserves (reserve_pixel_stage), synchronises and
// adds the times.
static int chunk_pixels(b200jpeg_encoder *e, const DecPlan &plan, int nk, uint8_t *pix, size_t row_pitch, size_t image_stride,
                        const std::vector<uint16_t> &qt, std::vector<uint32_t> &mt, const cudaEvent_t *ev)
{
  return plan.is_default && plan.nin != 4 ? idct_upsample_default(e, nk, pix, row_pitch, image_stride, ev)
                         : idct_upsample_opts(e, plan, nk, pix, row_pitch, image_stride, qt, mt, ev);
}

// The chunks of a batch: images in order until a chunk weighs about 1.6 M blocks (8 images of 3840x2160 4:2:0, 300 MB
// of coefficient and sample planes; an image heavier than that is a chunk of its own), or b200jpeg_encoder_set_chunk_images
// images.  Returns the first image of each chunk and n.
static std::vector<int> mixed_chunks(const b200jpeg_encoder *e, const std::vector<long long> &blocks)
{
  const int n = (int)blocks.size();
  std::vector<int> start(1, 0);
  long long acc = 0;
  for (int i = 0; i < n; i++) {
    const bool full = e->chunk_images_override > 0 ? i - start.back() == e->chunk_images_override : acc > 0 && acc + blocks[i] > 1600000LL;
    if (full) { start.push_back(i); acc = 0; }
    acc += blocks[i];
  }
  start.push_back(n);
  return start;
}

// the stages of the last decompress, appended to the stage times: the decode's, then the first `pixel` of "idct" and
// "upsample_color"
static void add_decompress_stage_times(b200jpeg_encoder *e, int pixel = 2)
{
  static const char *const extra[2] = {"idct", "upsample_color"};
  for (int k = 0; k < (e->dec_ms_prog ? 8 : 6); k++) { e->stage_names.push_back(kDecStages[k]); e->stage_ms.push_back(e->dec_ms[k < 6 ? k : k + 2]); e->stage_calls.push_back(1); }
  for (int k = 0; k < pixel; k++) { e->stage_names.push_back(extra[k]); e->stage_ms.push_back(e->dec_ms[6 + k]); e->stage_calls.push_back(1); }
}

// b200jpeg_decompress_yuv_batch: the entropy decode chunk by chunk, then per component the IDCT that
// tj3DecompressToYUVPlanes8 runs, stored straight into the planes (device planes), or into a compact staging buffer of
// the batch's written samples copied out with one cudaMemcpy2DAsync per plane and image (host planes)
static int decompress_yuv(b200jpeg_encoder *e, const b200jpeg_decompress_options *opts, const uint8_t *const *files, const size_t *sizes, int n,
                          uint8_t *const *planes, int planes_on_device, const size_t *plane_pitch, const size_t *plane_stride)
{
  if (!e || !opts || !files || !sizes || !planes || !plane_pitch || !plane_stride || n <= 0) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  // every refusal comes before any device work
  YuvPlan plan;
  b200jpeg_source_info s0;
  {
    static thread_local b200jpeg_source_info s;
    for (int i = 0; i < n; i++) {
      if (!files[i]) { set_error("image %d: no file", i); return B200JPEG_ERR_PARAM; }
      int rc = b200jpeg_parse_source(files[i], sizes[i], &s);
      YuvPlan pi;
      if (!rc) rc = plan_yuv(s, *opts, pi);
      if (!rc && s.data_precision != 8) { set_error("Unsupported JPEG data precision %d", s.data_precision); rc = B200JPEG_ERR_PARAM; }   // JERR_BAD_PRECISION
      if (!rc && s.sof == 0xC2 && !e->progressive_decode) { set_error("progressive (SOF2) source: only sequential files are decoded to planes unless progressive decode is on"); rc = B200JPEG_ERR_UNSUPPORTED; }
      if (rc) { std::string m = b200jpeg_last_error(); set_error("image %d: %s", i, m.c_str()); return rc; }
      if ((rc = check_tables_progression(s, i))) return rc;
      if (i == 0) { s0 = s; plan = pi; }
      bool same = s.image_width == s0.image_width && s.image_height == s0.image_height && s.num_components == s0.num_components;
      for (int c = 0; same && c < s.num_components; c++) same = s.h_samp_factor[c] == s0.h_samp_factor[c] && s.v_samp_factor[c] == s0.v_samp_factor[c];
      if (!same) { set_error("image %d: geometry (size, components, sampling) differs from image 0", i); return B200JPEG_ERR_PARAM; }
    }
  }
  const int nc = plan.nc;
  int cw[3], ch[3];                                        // the samples written: the IDCT output inside the plane
  for (int c = 0; c < nc; c++) {
    cw[c] = std::min(plan.iw[c], plan.pw[c]); ch[c] = std::min(plan.ih[c], plan.ph[c]);
    if (!planes[c]) { set_error("plane %d: no destination", c); return B200JPEG_ERR_PARAM; }
    if (plane_pitch[c] < (size_t)plan.pw[c] || (n > 1 && plane_stride[c] < plane_pitch[c] * (size_t)(plan.ph[c] - 1) + (size_t)plan.pw[c])) {
      set_error("plane %d: pitch %zu or stride %zu smaller than the plane (%dx%d)", c, plane_pitch[c], plane_stride[c], plan.pw[c], plan.ph[c]);
      return B200JPEG_ERR_PARAM;
    }
  }
  CU(cudaSetDevice(e->device));
  uint8_t *dst[3]; size_t dp[3], ds[3];
  if (planes_on_device) {
    for (int c = 0; c < nc; c++) { dst[c] = planes[c]; dp[c] = plane_pitch[c]; ds[c] = plane_stride[c]; }
  } else {
    size_t off[3], total = 0;
    for (int c = 0; c < nc; c++) { dp[c] = (size_t)cw[c]; ds[c] = dp[c] * ch[c]; off[c] = total; total += (ds[c] * n + 255) & ~(size_t)255; }
    if (int rc = e->d_dec_pixels.reserve(total)) return rc;
    for (int c = 0; c < nc; c++) dst[c] = e->d_dec_pixels.as<uint8_t>() + off[c];
  }
  while (e->pix_ev.size() < 2) { cudaEvent_t ev; CU(cudaEventCreate(&ev)); e->pix_ev.push_back(ev); }
  for (float &m : e->dec_ms) m = 0.f;
  e->dec_ms_prog = false;
  e->dec.want_markers = false;
  long long per = 0;
  for (int c = 0; c < nc; c++) per += (long long)(plan.iw[c] / plan.k) * (plan.ih[c] / plan.k);
  const std::vector<int> start = mixed_chunks(e, std::vector<long long>(n, per));
  e->chunk = 0;
  // the ifast multiplier tables: for the 8x8 ifast IDCT, and for 4:2:0 chroma at 1/2 under IFAST
  bool need_mt = plan.k == 8 && plan.method == B200JPEG_DCT_IFAST;
  for (int c = 0; c < nc; c++) need_mt |= plan.int_table[c];
  std::vector<uint16_t> qt;
  std::vector<uint32_t> mt;
  cudaStream_t s = e->stream;
  for (size_t j = 0; j + 1 < start.size(); j++) {
    const int i0 = start[j], nk = start[j + 1] - i0;
    e->chunk = std::max(e->chunk, nk);
    int rc = decode_files(e, files + i0, sizes + i0, nk, i0);
    if (rc) return rc;
    e->dec_ms_prog |= e->dec_prog;
    if ((rc = e->d_dec_quant.reserve((size_t)nk * nc * 128)) || (need_mt && (rc = e->d_dec_mtab.reserve((size_t)nk * nc * 256)))) return rc;
    if ((rc = upload_chunk_quant(e, nk, nc, qt))) return rc;
    if (need_mt) {
      mt.resize((size_t)nk * nc * 64);
      for (size_t t = 0; t < (size_t)nk * nc; t++) method_table(B200JPEG_DCT_IFAST, &qt[t * 64], &mt[t * 64]);
      CU(cudaMemcpyAsync(e->d_dec_mtab.p, mt.data(), mt.size() * 4, cudaMemcpyHostToDevice, s));
    }
    const DecGeom &g = e->dec.geom[0];
    CU(cudaEventRecord(e->pix_ev[0], s));
    for (int c = 0; c < nc; c++) {
      const bool by_mt = (plan.k == 8 && plan.method == B200JPEG_DCT_IFAST) || plan.int_table[c];
      const void *tab = by_mt ? static_cast<const void *>(e->d_dec_mtab.as<uint32_t>() + c * 64) : static_cast<const void *>(e->d_dec_quant.as<uint16_t>() + c * 64);
      const IdctDst d = {(long long)dp[c], (long long)ds[c], cw[c], ch[c]};
      launch_idct_plane(plan.k, plan.method, plan.int_table[c], reinterpret_cast<const int16_t *>(e->d_dec_planes.as<uint8_t>() + e->dec_plane_off[c]), tab, nc * 64,
                        dst[c] + (size_t)i0 * ds[c], d, g.wib[c], g.hib[c], nk, s);
    }
    CU(cudaEventRecord(e->pix_ev[1], s));
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(s));
    sum_decode_stage_times(e);
    float ms = 0.f; cudaEventElapsedTime(&ms, e->pix_ev[0], e->pix_ev[1]); e->dec_ms[6] += ms;
  }
  if (!planes_on_device) {
    for (int i = 0; i < n; i++)
      for (int c = 0; c < nc; c++)
        if (cw[c] > 0 && ch[c] > 0)
          CU(cudaMemcpy2DAsync(planes[c] + (size_t)i * plane_stride[c], plane_pitch[c], dst[c] + (size_t)i * ds[c], dp[c], cw[c], ch[c], cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
  }
  e->pending_marks = 0;
  e->stage_names.clear(); e->stage_ms.clear(); e->stage_calls.clear();
  add_decompress_stage_times(e, 1);
  return B200JPEG_OK;
}

// b200jpeg_decode_yuv_batch: host planes are staged into one compact device buffer (one cudaMemcpy2DAsync per plane
// and image), host pixels come back through one (one copy per image); then a single k_yuv_to_pixels launch
static int decode_yuv(b200jpeg_encoder *e, const b200jpeg_params *p, const uint8_t *const *planes, int planes_on_device, const size_t *plane_pitch,
                      const size_t *plane_stride, void *pixels, int pixels_on_device, size_t row_pitch, size_t image_stride, int n)
{
  if (!e || !p || !planes || !plane_pitch || !plane_stride || !pixels || n <= 0 || p->image_width <= 0 || p->image_height <= 0) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  if (p->data_precision != 8) { set_error("data_precision %d: YUV planes are decoded at 8 bits", p->data_precision); return B200JPEG_ERR_PARAM; }
  const int cs = p->in_color_space, nc = p->num_components, W = p->image_width, H = p->image_height;
  if (cs == B200JPEG_CS_CMYK) { set_error("Cannot decode YUV images into packed-pixel CMYK images."); return B200JPEG_ERR_PARAM; }
  if (cs != B200JPEG_CS_GRAYSCALE && !B200JPEG_CS_IS_RGB(cs)) { set_error("in_color_space %d is not a TurboJPEG pixel format", cs); return B200JPEG_ERR_PARAM; }
  // the TJSAMP_* the planes are in: gray, or YCbCr with component 0 at 1, 2 or 4 each way (as tj3_params sets them) over 1x1 chroma
  const b200jpeg_component_info *ci = p->comp_info;
  const int h0 = ci[0].h_samp_factor, v0 = ci[0].v_samp_factor;
  bool known = (nc == 1 && p->jpeg_color_space == B200JPEG_CS_GRAYSCALE) ||
               (nc == 3 && p->jpeg_color_space == B200JPEG_CS_YCbCr && ci[1].h_samp_factor == 1 && ci[1].v_samp_factor == 1 && ci[2].h_samp_factor == 1 &&
                ci[2].v_samp_factor == 1 && ((h0 == 1 && v0 == 1) || (h0 == 2 && v0 == 1) || (h0 == 2 && v0 == 2) || (h0 == 1 && v0 == 2) || (h0 == 4 && v0 == 1) || (h0 == 1 && v0 == 4)));
  if (!known) { set_error("TJPARAM_SUBSAMP must be specified (the parameter block's components and sampling name no TJSAMP_* layout)"); return B200JPEG_ERR_PARAM; }
  const int ps = cs == B200JPEG_CS_GRAYSCALE ? 1 : B200JPEG_CS_PIXELSIZE(cs);
  if (row_pitch < (size_t)W * ps || (n > 1 && image_stride < row_pitch * (size_t)(H - 1) + (size_t)W * ps)) { set_error("row_pitch or image_stride smaller than the image (%dx%d, %d bytes a pixel)", W, H, ps); return B200JPEG_ERR_PARAM; }
  YuvPix d; memset(&d, 0, sizeof d);
  d.ps = ps; d.hs = h0 == 4 ? 2 : h0 - 1; d.vs = v0 == 4 ? 2 : v0 - 1;
  d.conv = cs == B200JPEG_CS_GRAYSCALE ? UPS_GRAY : nc == 1 ? UPS_GRAY_RGB : UPS_YCC_RGB;
  if (ps > 1) {
    const int f = B200JPEG_CS_FIRST(cs), bf = B200JPEG_CS_BLUE_FIRST(cs);
    d.off[0] = f + (bf ? 2 : 0); d.off[1] = f + 1; d.off[2] = f + (bf ? 0 : 2); d.off[3] = f ? 0 : 3;
  }
  const int nread = d.conv == UPS_YCC_RGB ? 3 : 1;           // a gray pixel format reads luma only
  int pw[3], ph[3];
  for (int c = 0; c < nread; c++) {
    b200jpeg_yuv_plane_dims(p, c, &pw[c], &ph[c]);
    if (!planes[c]) { set_error("plane %d: no source", c); return B200JPEG_ERR_PARAM; }
    if (plane_pitch[c] < (size_t)pw[c] || (n > 1 && plane_stride[c] < plane_pitch[c] * (size_t)(ph[c] - 1) + (size_t)pw[c])) {
      set_error("plane %d: pitch %zu or stride %zu smaller than the plane (%dx%d)", c, plane_pitch[c], plane_stride[c], pw[c], ph[c]);
      return B200JPEG_ERR_PARAM;
    }
  }
  CU(cudaSetDevice(e->device));
  cudaStream_t s = e->stream;
  size_t off[3], total = 0;
  for (int c = 0; c < nread; c++) { off[c] = total; total += ((size_t)pw[c] * ph[c] * n + 255) & ~(size_t)255; }
  int rc;
  if (!planes_on_device && (rc = e->d_dec_samples.reserve(total))) return rc;
  const size_t dp = ((size_t)W * ps + 3) & ~(size_t)3, ds = dp * H;
  if (!pixels_on_device && (rc = e->d_dec_pixels.reserve(ds * (size_t)n))) return rc;
  while (e->pix_ev.size() < 2) { cudaEvent_t ev; CU(cudaEventCreate(&ev)); e->pix_ev.push_back(ev); }
  for (int c = 0; c < nread; c++) {
    if (planes_on_device) { d.plane[c] = planes[c]; d.pitch[c] = (long long)plane_pitch[c]; d.stride[c] = (long long)plane_stride[c]; continue; }
    uint8_t *st = e->d_dec_samples.as<uint8_t>() + off[c];
    d.plane[c] = st; d.pitch[c] = pw[c]; d.stride[c] = (long long)pw[c] * ph[c];
    for (int i = 0; i < n; i++)
      CU(cudaMemcpy2DAsync(st + (size_t)i * d.stride[c], pw[c], planes[c] + (size_t)i * plane_stride[c], plane_pitch[c], pw[c], ph[c], cudaMemcpyHostToDevice, s));
  }
  uint8_t *pix = pixels_on_device ? static_cast<uint8_t *>(pixels) : e->d_dec_pixels.as<uint8_t>();
  CU(cudaEventRecord(e->pix_ev[0], s));
  launch_yuv_to_pixels(d, pix, pixels_on_device ? row_pitch : dp, pixels_on_device ? image_stride : ds, W, H, n, s);
  CU(cudaEventRecord(e->pix_ev[1], s));
  CU(cudaGetLastError());
  if (!pixels_on_device)
    for (int i = 0; i < n; i++)
      CU(cudaMemcpy2DAsync(static_cast<uint8_t *>(pixels) + (size_t)i * image_stride, row_pitch, pix + (size_t)i * ds, dp, (size_t)W * ps, H, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  float ms = 0.f; cudaEventElapsedTime(&ms, e->pix_ev[0], e->pix_ev[1]);
  e->pending_marks = 0;
  e->stage_names.clear(); e->stage_ms.clear(); e->stage_calls.clear();
  e->stage_names.push_back("yuv_to_pixels"); e->stage_ms.push_back(ms); e->stage_calls.push_back(1);
  return B200JPEG_OK;
}

// the stage times of the last encode added into (names, ms, calls)
static void merge_stage_times(const b200jpeg_encoder *e, std::vector<const char *> &names, std::vector<float> &ms, std::vector<int> &calls)
{
  for (size_t k = 0; k < e->stage_names.size(); k++) {
    size_t j = 0;
    while (j < names.size() && strcmp(names[j], e->stage_names[k])) j++;
    if (j == names.size()) { names.push_back(e->stage_names[k]); ms.push_back(0.f); calls.push_back(0); }
    ms[j] += e->stage_ms[k]; calls[j] += e->stage_calls[k];
  }
}

// ------------------------------------------------------------------- decompress and recompress from JPEG files
// Every call that decodes files to pixels (b200jpeg_decompress_batch, _renditions and _mixed, and the recompress forms
// of each) runs through one checker (plan_rungs), one per-chunk loop (mixed_files) and one chunk rule (mixed_chunks).
// A single call is one rung; the single and rendition calls also hold every file to image 0's geometry.  The entropy
// decode takes the files as they come (DecBatch::mixed); the pixel stage of a chunk of one geometry with evenly spaced
// outputs is the one-geometry route (chunk_pixels), of every other chunk the ragged IDCT and upsampling kernels driven
// by a work table, so a chunk costs the same launches whatever the mix of sizes.
//
// Refusals come before any device work, in this order: the arguments, the sources image by image, the rungs' options,
// then the output buffers, or each parameter block (b200jpeg_validate, precision, its image's decoded geometry).  The
// sources come before the parameter blocks because a caller that cannot build an image's block from a refused file
// passes an empty one and relies on the file's own refusal (Encoder.recompress_mixed).

// A per-rung, per-image array of a call, read as a[r * rung_step + i * image_step]: a mixed call passes one entry per
// output, a rendition call one per rung (image step 0), a single call one in all (both steps 0).
template <class T> struct View {
  const T *a; size_t rung_step, image_step;
  const T &operator()(int r, int i) const { return a[(size_t)r * rung_step + (size_t)i * image_step]; }
};

// A decompress or recompress call: its kind, its R rungs' options and its n files.  The kind decides whether the files
// must share one geometry (single and rendition calls) and how messages name a rung and an image: a single call names
// neither, a rendition call the rung, a mixed call the rung and the image.
enum CallKind { SINGLE_CALL, RENDITION_CALL, MIXED_CALL };
struct Call {
  CallKind kind; int R, n;
  const b200jpeg_decompress_options *opts;
  const uint8_t *const *files; const size_t *sizes;
};

// the front of a message about image i of rung r (i < 0: about the rung as a whole)
static std::string where(const Call &c, int r, int i)
{
  char b[64] = "";
  if (c.kind == MIXED_CALL && i >= 0) snprintf(b, sizeof b, "rendition %d, image %d: ", r, i);
  else if (c.kind != SINGLE_CALL) snprintf(b, sizeof b, "rendition %d: ", r);
  return b;
}

// What a call knows before any device work: each image's chunk weight, the distinct option sets of the rungs (set[r]:
// rung r's; first[k]: the first rung of set k) and each set's plan for each image.
struct RungSets {
  std::vector<long long> weight;
  std::vector<int> set, first;
  std::vector<std::vector<DecPlan>> plan;              // [set][image]
};

// what a one-geometry chunk's single conversion needs its images to share beyond the geometry: RGB-coded or not for
// three components, YCCK or CMYK for four
static int conversion_class(const b200jpeg_source_info &s)
{
  return (s.num_components == 3 && s.jpeg_color_space == B200JPEG_CS_RGB) || (s.num_components == 4 && s.jpeg_color_space == B200JPEG_CS_YCCK);
}

// The checks of a call's sources and rung options: each file parsed into one scratch header and checked as
// b200jpeg_decompress_batch takes it, then each distinct option set planned for it.  A refused option set is reported
// after every source passed, for the first image it fails on, naming the image only when that is not image 0.
static int plan_rungs(const b200jpeg_encoder *e, const Call &c, RungSets &m)
{
  m = RungSets();
  for (int r = 0; r < c.R; r++) {
    const b200jpeg_decompress_options &o = c.opts[r];
    int k = 0;
    for (; k < (int)m.first.size(); k++) {
      const b200jpeg_decompress_options &f = c.opts[m.first[k]];
      if (f.scale_num == o.scale_num && f.scale_denom == o.scale_denom && f.dct_method == o.dct_method &&
          f.do_fancy_upsampling == o.do_fancy_upsampling && f.out_color_space == o.out_color_space && f.all_scales == o.all_scales &&
          f.cmyk == o.cmyk) break;
    }
    if (k == (int)m.first.size()) m.first.push_back(r);
    m.set.push_back(k);
  }
  bool cmyk = true;                                    // 4-component sources: only when every rung decodes them
  for (int r = 0; r < c.R; r++) cmyk &= c.opts[r].cmyk != 0;
  const int K = (int)m.first.size();
  m.plan.assign(K, std::vector<DecPlan>(c.n));
  m.weight.assign(c.n, 0);
  std::vector<int> bad(K, -1), bad_rc(K, 0);           // per set: the first image whose plan was refused, and the code
  std::vector<std::string> why(K);
  static thread_local b200jpeg_source_info s;
  std::array<int, 12> g0{};
  for (int i = 0; i < c.n; i++) {
    if (!c.files[i]) { set_error("image %d: no file", i); return B200JPEG_ERR_PARAM; }
    int rc = b200jpeg_parse_source(c.files[i], c.sizes[i], &s);
    if (rc) { std::string msg = b200jpeg_last_error(); set_error("image %d: %s", i, msg.c_str()); return rc; }
    if ((rc = check_decompress_source(s, i, e->progressive_decode, cmyk))) return rc;
    // the geometry one-geometry calls compare: size, components, sampling factors, and the conversion class
    const int nc = s.num_components;
    std::array<int, 12> g{s.image_width, s.image_height, nc, conversion_class(s)};
    int hmax = 1, vmax = 1;
    for (int ch = 0; ch < nc; ch++) {
      g[4 + 2 * ch] = s.h_samp_factor[ch]; g[5 + 2 * ch] = s.v_samp_factor[ch];
      hmax = std::max(hmax, s.h_samp_factor[ch]); vmax = std::max(vmax, s.v_samp_factor[ch]);
    }
    if (i == 0) g0 = g;
    if (c.kind != MIXED_CALL && g != g0) { set_error("image %d: geometry (size, components, sampling, colour space) differs from image 0", i); return B200JPEG_ERR_PARAM; }
    // the chunk weight: the image's blocks, those whose IDCT writes more than 8 x 8 samples counted as ssize^2 / 64
    // blocks under the largest of the sets' plans, so a chunk's sample planes stay the size they have at 1/1 (DESIGN §14)
    for (int k = 0; k < K; k++) {
      if (bad[k] >= 0) continue;
      const DecPlan &p = m.plan[k][i];
      if ((rc = plan_decompress(s, c.opts[m.first[k]], m.plan[k][i]))) { bad[k] = i; bad_rc[k] = rc; why[k] = b200jpeg_last_error(); continue; }
      long long w = 0;
      for (int ch = 0; ch < nc; ch++)
        w += (long long)div_up((long long)s.image_width * s.h_samp_factor[ch], hmax * 8) * div_up((long long)s.image_height * s.v_samp_factor[ch], vmax * 8) *
             std::max(64, p.ssize[ch] * p.ssize[ch]) / 64;
      m.weight[i] = std::max(m.weight[i], w);
    }
  }
  for (int k = 0; k < K; k++)
    if (bad[k] >= 0) { set_error("%s%s", where(c, m.first[k], bad[k] ? bad[k] : -1).c_str(), why[k].c_str()); return bad_rc[k]; }
  return B200JPEG_OK;
}

// where image i of a pixel output goes
struct MixedOut { uint8_t *pix; size_t row_pitch; };

// One option set's pixel stage of a mixed chunk, staged on the host: the IDCT launches (one per component slot and
// IDCT size present among the images), the upsampling launch, and the bytes of their descriptors and work tables.
struct MixLaunch { int c, size; size_t desc, work; unsigned ncta; };
struct MixStage {
  std::vector<uint8_t> meta;
  std::vector<MixLaunch> idct;
  size_t ups_desc = 0, ups_work = 0; unsigned ups_cta = 0;         // 1- and 3-component images
  size_t ups4_desc = 0, ups4_work = 0; unsigned ups4_cta = 0;      // 4-component images
  bool need_mt = false;
};

template <class T> static size_t meta_put(std::vector<uint8_t> &m, const T *p, size_t count)
{
  const size_t off = (m.size() + 15) & ~(size_t)15;
  m.resize(off + count * sizeof(T));
  if (count) memcpy(m.data() + off, p, count * sizeof(T));
  return off;
}

// the bytes of one set's sample planes in a chunk (images [i0, i0 + nk)); soff[i][c]: where image i's plane c starts
static size_t mixed_sample_layout(const DecBatch &b, const std::vector<DecPlan> &plan, int i0, int nk, std::vector<std::array<size_t, 4>> &soff)
{
  size_t total = 0;
  soff.assign(nk, std::array<size_t, 4>{0, 0, 0, 0});
  for (int i = 0; i < nk; i++) {
    const DecGeom &g = b.geom[i]; const DecPlan &p = plan[i0 + i];
    for (int c = 0; c < g.nc; c++) {
      if (!p.needed[c]) continue;
      soff[i][c] = total; total += ((size_t)g.wib[c] * g.hib[c] * p.ssize[c] * p.ssize[c] + 255) & ~(size_t)255;
    }
  }
  return total;
}

static void stage_mixed(const b200jpeg_encoder *e, const std::vector<DecPlan> &plan, int i0, int nk, int qs, const MixedOut *out, uint8_t *samples, MixStage &st)
{
  const DecBatch &b = e->dec;
  std::vector<std::array<size_t, 4>> soff;
  mixed_sample_layout(b, plan, i0, nk, soff);
  st = MixStage();
  std::vector<IdctImg> d; std::vector<uint32_t> w;
  for (int c = 0; c < 4; c++)
    for (int size = 1; size <= 16; size++) {
      d.clear(); w.clear();
      const int bpc = idct_blocks_per_cta(size);
      for (int i = 0; i < nk; i++) {
        const DecGeom &g = b.geom[i]; const DecPlan &p = plan[i0 + i];
        if (c >= g.nc || !p.needed[c] || p.ssize[c] != size) continue;
        st.need_mt |= size == 8 && p.method != B200JPEG_DCT_ISLOW;
        IdctImg im;
        im.coef = g.base[c]; im.out = (long long)soff[i][c]; im.wib = g.wib[c]; im.hib = g.hib[c]; im.tab = (i * qs + c) * 64; im.cta0 = (int)w.size();
        const long long ncta = ((long long)g.wib[c] * g.hib[c] + bpc - 1) / bpc;
        w.insert(w.end(), (size_t)ncta, (uint32_t)d.size());
        d.push_back(im);
      }
      if (d.empty()) continue;
      MixLaunch l;
      l.c = c; l.size = size; l.ncta = (unsigned)w.size();
      l.desc = meta_put(st.meta, d.data(), d.size()); l.work = meta_put(st.meta, w.data(), w.size());
      st.idct.push_back(l);
    }
  // the upsampling images, 4-component ones in a table of their own for k_upsample_ragged<4>
  std::vector<UpsImg> u; std::vector<UpsImg4> u4; std::vector<uint32_t> w4; w.clear();
  for (int i = 0; i < nk; i++) {
    const DecGeom &g = b.geom[i]; const DecPlan &p = plan[i0 + i];
    UpsImg4 im; memset(&im, 0, sizeof im);
    for (int c = 0; c < g.nc; c++)
      if (p.needed[c]) ups_component(im.o, p, c, samples + soff[i][c], g.wib[c] * p.ssize[c], 0);
    ups_conversion(im.o, p);
    im.pix = out[i].pix; im.row_pitch = (long long)out[i].row_pitch; im.W = p.out_w; im.H = p.out_h;
    im.gx = div_up(p.out_w, 64);
    if (p.nin == 4) {
      im.cta0 = (int)w4.size();
      w4.insert(w4.end(), (size_t)im.gx * div_up(p.out_h, 4), (uint32_t)u4.size());
      u4.push_back(im);
      continue;
    }
    UpsImg im3;
    memset(&im3, 0, sizeof im3);
    im3.o = ups_narrow(im.o); im3.pix = im.pix; im3.row_pitch = im.row_pitch; im3.W = im.W; im3.H = im.H; im3.gx = im.gx; im3.cta0 = (int)w.size();
    w.insert(w.end(), (size_t)im3.gx * div_up(p.out_h, 4), (uint32_t)u.size());
    u.push_back(im3);
  }
  st.ups_cta = (unsigned)w.size();
  st.ups_desc = meta_put(st.meta, u.data(), u.size()); st.ups_work = meta_put(st.meta, w.data(), w.size());
  st.ups4_cta = (unsigned)w4.size();
  st.ups4_desc = meta_put(st.meta, u4.data(), u4.size()); st.ups4_work = meta_put(st.meta, w4.data(), w4.size());
}

// whether images [i0, i0 + nk) of a set's outputs lie one image stride apart at one row pitch (stride: that stride)
static bool evenly_spaced(const std::vector<MixedOut> &o, int i0, int nk, size_t &stride)
{
  stride = nk > 1 ? (size_t)(o[i0 + 1].pix - o[i0].pix) : 0;
  for (int i = 1; i < nk; i++)
    if (o[i0 + i].pix < o[i0].pix || o[i0 + i].pix != o[i0].pix + (size_t)i * stride || o[i0 + i].row_pitch != o[i0].row_pitch) return false;
  return true;
}

// jpeg_read_scanlines for a call's files, to every option set's outputs (out[k][i]): per chunk the entropy decode, then
// each set's pixel stage, enqueued together and synchronised once.  A chunk of one geometry (size, sampling,
// components, RGB-coded or not) whose outputs are evenly spaced takes the one-geometry route (chunk_pixels), faster in
// its upsampling (DESIGN §12); every other chunk the ragged one.
static int mixed_files(b200jpeg_encoder *e, const Call &c, const RungSets &m, const std::vector<std::vector<MixedOut>> &out, bool want_markers)
{
  const int K = (int)m.first.size(), n = c.n;
  while (e->pix_ev.size() < (size_t)K * 3) { cudaEvent_t ev; CU(cudaEventCreate(&ev)); e->pix_ev.push_back(ev); }
  for (float &ms : e->dec_ms) ms = 0.f;
  e->dec_ms_prog = false;
  e->dec.want_markers = want_markers;
  if (want_markers) e->dec_markers.assign(n, std::vector<uint8_t>());
  const std::vector<int> start = mixed_chunks(e, m.weight);
  e->chunk = 0;
  std::vector<uint16_t> qt; std::vector<uint32_t> mt; std::vector<MixStage> st(K);
  std::vector<std::array<size_t, 4>> soff;
  cudaStream_t s = e->stream;
  for (size_t ch = 0; ch + 1 < start.size(); ch++) {
    const int i0 = start[ch], nk = start[ch + 1] - i0;
    e->chunk = std::max(e->chunk, nk);
    int rc = decode_files(e, c.files + i0, c.sizes + i0, nk, i0, true);
    if (rc) return rc;
    e->dec_ms_prog |= e->dec_prog;
    if (want_markers) for (int i = 0; i < nk; i++) e->dec_markers[i0 + i].swap(e->dec.markers[i]);
    const DecGeom &g0 = e->dec.geom[0];
    bool one = true;
    int qs = 1;                                          // components per image in the chunk's table layout [nk][qs][64]
    for (int i = 0; i < nk; i++) {
      const DecGeom &g = e->dec.geom[i];
      qs = std::max(qs, g.nc);
      one &= g.W == g0.W && g.H == g0.H && g.nc == g0.nc && conversion_class(e->dec.info[i]) == conversion_class(e->dec.info[0]);
      for (int c = 0; c < g.nc; c++) one &= g.h[c] == g0.h[c] && g.v[c] == g0.v[c];
    }
    std::vector<size_t> stride(K, 0);
    std::vector<char> uniform(K, 0);
    for (int k = 0; k < K; k++) uniform[k] = one && evenly_spaced(out[k], i0, nk, stride[k]);
    // every buffer the chunk's pixel stages use is reserved before the first is enqueued
    size_t samples = 0, meta = 0;
    for (int k = 0; k < K; k++)
      if (uniform[k]) { if ((rc = reserve_pixel_stage(e, m.plan[k][i0], nk))) return rc; }
      else samples = std::max(samples, mixed_sample_layout(e->dec, m.plan[k], i0, nk, soff));
    if ((rc = e->d_dec_samples.reserve(samples)) || (rc = e->d_dec_quant.reserve((size_t)nk * qs * 128)) || (rc = e->d_dec_mtab.reserve((size_t)nk * qs * 256))) return rc;
    for (int k = 0; k < K; k++)
      if (!uniform[k]) { stage_mixed(e, m.plan[k], i0, nk, qs, out[k].data() + i0, e->d_dec_samples.as<uint8_t>(), st[k]); meta = std::max(meta, st[k].meta.size()); }
    if ((rc = e->d_mix_meta.reserve(meta))) return rc;
    if ((rc = upload_chunk_quant(e, nk, qs, qt))) return rc;
    const int16_t *coef[4];
    for (int c = 0; c < 4; c++) coef[c] = reinterpret_cast<const int16_t *>(e->d_dec_planes.as<uint8_t>() + e->dec_plane_off[c]);
    for (int k = 0; k < K; k++) {
      const MixStage &g = st[k];
      const int method = m.plan[k][i0].method;
      const cudaEvent_t *ev = &e->pix_ev[(size_t)k * 3];
      if (uniform[k]) {
        const MixedOut &o = out[k][i0];
        if ((rc = chunk_pixels(e, m.plan[k][i0], nk, o.pix, o.row_pitch, stride[k], qt, mt, ev))) return rc;
        continue;
      }
      // stream order keeps these uploads behind the previous set's kernels, which read the same buffers
      if (g.need_mt) {
        mt.resize(qt.size());
        for (size_t t = 0; t < (size_t)nk * qs; t++) method_table(method, &qt[t * 64], &mt[t * 64]);
        CU(cudaMemcpyAsync(e->d_dec_mtab.p, mt.data(), mt.size() * 4, cudaMemcpyHostToDevice, s));
      }
      CU(cudaMemcpyAsync(e->d_mix_meta.p, g.meta.data(), g.meta.size(), cudaMemcpyHostToDevice, s));
      const uint8_t *meta_d = e->d_mix_meta.as<uint8_t>();
      CU(cudaEventRecord(ev[0], s));
      for (const MixLaunch &l : g.idct) {
        const bool by_method = l.size == 8 && method != B200JPEG_DCT_ISLOW;
        const void *tab = by_method ? static_cast<const void *>(e->d_dec_mtab.as<uint32_t>()) : static_cast<const void *>(e->d_dec_quant.as<uint16_t>());
        launch_idct_ragged(l.size, method, coef[l.c], tab, e->d_dec_samples.as<uint8_t>(), reinterpret_cast<const uint32_t *>(meta_d + l.work),
                           reinterpret_cast<const IdctImg *>(meta_d + l.desc), l.ncta, s);
      }
      CU(cudaEventRecord(ev[1], s));
      if (g.ups_cta) launch_upsample_ragged(reinterpret_cast<const uint32_t *>(meta_d + g.ups_work), reinterpret_cast<const UpsImg *>(meta_d + g.ups_desc), g.ups_cta, s);
      if (g.ups4_cta) launch_upsample_ragged(reinterpret_cast<const uint32_t *>(meta_d + g.ups4_work), reinterpret_cast<const UpsImg4 *>(meta_d + g.ups4_desc), g.ups4_cta, s);
      CU(cudaEventRecord(ev[2], s));
      CU(cudaGetLastError());
    }
    CU(cudaStreamSynchronize(s));
    sum_decode_stage_times(e);
    for (int k = 0; k < K; k++)
      for (int j = 0; j < 2; j++) { float ms = 0.f; cudaEventElapsedTime(&ms, e->pix_ev[(size_t)k * 3 + j], e->pix_ev[(size_t)k * 3 + j + 1]); e->dec_ms[6 + j] += ms; }
  }
  return B200JPEG_OK;
}

// each set's pixels for the whole batch in one device buffer, the images in order[k], each row the decoded row padded
// to 4 bytes (the pitch the encoder reads)
static int reserve_set_pixels(b200jpeg_encoder *e, const RungSets &m, const std::vector<std::vector<int>> &order, std::vector<std::vector<MixedOut>> &out)
{
  const int K = (int)m.first.size(), n = (int)m.weight.size();
  if ((int)e->d_rend_pixels.size() < K) e->d_rend_pixels.resize(K);
  out.assign(K, std::vector<MixedOut>(n));
  std::vector<size_t> off(n);
  for (int k = 0; k < K; k++) {
    size_t total = 0;
    for (int i : order[k]) {
      const DecPlan &p = m.plan[k][i];
      out[k][i].row_pitch = ((size_t)p.out_w * p.out_nc + 3) & ~(size_t)3; off[i] = total; total += out[k][i].row_pitch * p.out_h;
    }
    if (int rc = e->d_rend_pixels[k].reserve(total)) return rc;
    for (int i = 0; i < n; i++) out[k][i].pix = e->d_rend_pixels[k].as<uint8_t>() + off[i];
  }
  return B200JPEG_OK;
}

// The decompress calls: image i of rung r goes to pix(r, i) + i * stride(r, i), rows pitch(r, i) apart.  One decode per
// chunk and one pixel stage per distinct option set; on the device the first rung of each set receives its pixels in
// place, every other output is copied from its set's.
static int decompress_rungs(b200jpeg_encoder *e, const Call &c, View<void *> pix, View<size_t> pitch, View<size_t> stride, int on_device)
{
  RungSets m;
  int rc = plan_rungs(e, c, m);
  if (rc) return rc;
  const int n = c.n, K = (int)m.first.size();
  for (int r = 0; r < c.R; r++)
    for (int i = 0; i < n; i++) {
      const DecPlan &p = m.plan[m.set[r]][i];
      const size_t row = (size_t)p.out_w * p.out_nc;
      if (c.kind == MIXED_CALL && (!pix(r, i) || pitch(r, i) < row)) {
        set_error("rendition %d, image %d: no pixel buffer, or row_pitch smaller than the decoded row (%dx%d, %d components)", r, i, p.out_w, p.out_h, p.out_nc);
        return B200JPEG_ERR_PARAM;
      }
      if (c.kind != MIXED_CALL && (!pix(r, i) || pitch(r, i) < row || (n > 1 && stride(r, i) < pitch(r, i) * (size_t)(p.out_h - 1) + row))) {
        set_error("%s%srow_pitch or image_stride smaller than the decoded image (%dx%d, %d components)", where(c, r, -1).c_str(),
                  c.kind == RENDITION_CALL ? "no pixel buffer, or " : "", p.out_w, p.out_h, p.out_nc);
        return B200JPEG_ERR_PARAM;
      }
    }
  CU(cudaSetDevice(e->device));
  auto dst = [&](int r, int i) { return static_cast<uint8_t *>(pix(r, i)) + (size_t)i * stride(r, i); };
  std::vector<std::vector<MixedOut>> out(K, std::vector<MixedOut>(n));
  if (on_device) {
    for (int k = 0; k < K; k++)
      for (int i = 0; i < n; i++) out[k][i] = MixedOut{dst(m.first[k], i), pitch(m.first[k], i)};
  } else {
    std::vector<std::vector<int>> order(K, std::vector<int>(n));
    for (std::vector<int> &o : order) for (int i = 0; i < n; i++) o[i] = i;
    if ((rc = reserve_set_pixels(e, m, order, out))) return rc;
  }
  if ((rc = mixed_files(e, c, m, out, false))) return rc;
  for (int r = 0; r < c.R; r++) {
    const int k = m.set[r];
    if (on_device && r == m.first[k]) continue;
    for (int i = 0; i < n; i++) {
      const DecPlan &p = m.plan[k][i];
      CU(cudaMemcpy2DAsync(dst(r, i), pitch(r, i), out[k][i].pix, out[k][i].row_pitch, (size_t)p.out_w * p.out_nc, p.out_h,
                           on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, e->stream));
    }
  }
  CU(cudaStreamSynchronize(e->stream));
  e->pending_marks = 0;
  e->stage_names.clear(); e->stage_ms.clear(); e->stage_calls.clear();
  add_decompress_stage_times(e);
  return B200JPEG_OK;
}

// The recompress calls: image i of rung r is encoded with params(r, i).  The pixels of each distinct option set as
// decompress_rungs makes them, then per rung one encode per group of images with identical parameter blocks (one
// decoded size, so one pitch and stride), from the group's images one after another; outputs numbered rung by rung in
// input order.
static int recompress_rungs(b200jpeg_encoder *e, const Call &c, View<b200jpeg_params> params)
{
  const int n = c.n, R = c.R;
  const bool mixed = c.kind == MIXED_CALL;
  RungSets m;
  int rc = plan_rungs(e, c, m);
  if (rc) return rc;
  // group[r][i]: the first image of rung r whose parameter block equals image i's
  std::vector<std::vector<int>> group(R, std::vector<int>(n));
  for (int r = 0; r < R; r++)
    for (int i = 0; i < n; i++) {
      const b200jpeg_params *p = &params(r, i);
      if (i == 0 || params.image_step) {
        if ((rc = b200jpeg_validate(p))) { std::string msg = b200jpeg_last_error(); set_error("%s%s", where(c, r, i).c_str(), msg.c_str()); return rc; }
        if (p->data_precision != 8) {
          set_error("%sthe source%s to 8-bit samples, the parameter block has data_precision %d", where(c, r, i).c_str(), mixed ? " decodes" : "s decode", p->data_precision);
          return B200JPEG_ERR_PARAM;
        }
      }
      const DecPlan &pl = m.plan[m.set[r]][i];
      if (pl.out_w != p->image_width || pl.out_h != p->image_height || pl.out_cs != p->in_color_space || pl.out_nc != p->input_components) {
        set_error("%sthe source%s to %dx%d pixels of %d samples in colour space %d, the parameter block describes %dx%d of %d in %d (see b200jpeg_decompress_output%s)",
                  where(c, r, i).c_str(), mixed ? " decodes" : "s decode", pl.out_w, pl.out_h, pl.out_nc, pl.out_cs, p->image_width, p->image_height,
                  p->input_components, p->in_color_space, c.kind == SINGLE_CALL ? "" : "_opts");
        return B200JPEG_ERR_PARAM;
      }
      int g = 0;
      while (g < i && !(group[r][g] == g && (&params(r, g) == p || !memcmp(&params(r, g), p, sizeof *p)))) g++;
      group[r][i] = g;
    }
  CU(cudaSetDevice(e->device));
  // each set's buffer holds the images group by group as its first rung forms them, so that rung encodes in place
  const int K = (int)m.first.size();
  std::vector<std::vector<int>> order(K);
  for (int k = 0; k < K; k++) {
    const std::vector<int> &gr = group[m.first[k]];
    for (int g = 0; g < n; g++) if (gr[g] == g) for (int i = g; i < n; i++) if (gr[i] == g) order[k].push_back(i);
  }
  std::vector<std::vector<MixedOut>> out;
  if ((rc = reserve_set_pixels(e, m, order, out))) return rc;
  if ((rc = mixed_files(e, c, m, out, true))) return rc;
  // a group's files move to e->rend_files when another encode follows and would reuse the file arenas; the last
  // encode's stay where they are.  kept: per output, (offset in rend_files, size), or (SIZE_MAX, its index in the last
  // encode).
  int last = n - 1;
  while (group[R - 1][last] != last) last--;
  std::vector<std::pair<size_t, size_t>> kept((size_t)R * n);
  std::vector<const char *> names; std::vector<float> ms; std::vector<int> calls;
  std::vector<std::vector<uint8_t>> markers;
  size_t scan_bytes = 0;
  e->rend_files.clear();
  for (int r = 0; r < R; r++) {
    const int k = m.set[r];
    for (int g = 0; g < n; g++) {
      if (group[r][g] != g) continue;
      std::vector<int> mem;
      for (int i = g; i < n; i++) if (group[r][i] == g) mem.push_back(i);
      const size_t pitch = out[k][g].row_pitch, stride = pitch * (size_t)m.plan[k][g].out_h;
      bool in_place = true;
      for (size_t j = 1; j < mem.size(); j++) in_place &= out[k][mem[j]].pix == out[k][mem[0]].pix + j * stride;
      const uint8_t *src = out[k][mem[0]].pix;
      if (!in_place) {                                 // another rung's grouping: gather the group's images
        if ((rc = e->d_dec_pixels.reserve(stride * mem.size()))) return rc;
        for (size_t j = 0; j < mem.size(); j++)
          CU(cudaMemcpyAsync(e->d_dec_pixels.as<uint8_t>() + j * stride, out[k][mem[j]].pix, stride, cudaMemcpyDeviceToDevice, e->stream));
        src = e->d_dec_pixels.as<uint8_t>();
      }
      const std::vector<std::vector<uint8_t>> *mk = &e->dec_markers;     // the whole batch in input order
      if ((int)mem.size() < n) {
        markers.resize(mem.size());
        for (size_t j = 0; j < mem.size(); j++) markers[j] = e->dec_markers[mem[j]];
        mk = &markers;
      }
      if ((rc = encode_common(e, &params(r, g), src, 1, pitch, stride, (int)mem.size(), false, nullptr, nullptr, mk))) return rc;
      scan_bytes += e->last_scan_bytes;
      merge_stage_times(e, names, ms, calls);
      const bool final = r + 1 == R && g == last;
      for (size_t j = 0; j < mem.size(); j++) {
        kept[(size_t)r * n + mem[j]] = final ? std::make_pair(SIZE_MAX, j) : std::make_pair(e->rend_files.size(), e->files[j].second);
        if (!final) e->rend_files.insert(e->rend_files.end(), e->files[j].first, e->files[j].first + e->files[j].second);
      }
    }
  }
  const std::vector<std::pair<uint8_t *, size_t>> fin(e->files);
  e->files.clear();
  for (const std::pair<size_t, size_t> &f : kept) e->files.push_back(f.first == SIZE_MAX ? fin[f.second] : std::make_pair(e->rend_files.data() + f.first, f.second));
  e->last_scan_bytes = scan_bytes;
  e->stage_names = names; e->stage_ms = ms; e->stage_calls = calls;
  add_decompress_stage_times(e);
  return B200JPEG_OK;
}

}  // namespace b200

extern "C" {

int b200jpeg_decompress_batch(b200jpeg_encoder *e, const uint8_t *const *files, const size_t *sizes, int n_images,
                              void *pixels, int pixels_on_device, size_t row_pitch, size_t image_stride)
{
  const b200jpeg_decompress_options o = b200jpeg_default_decompress_options();
  return b200jpeg_decompress_batch_opts(e, &o, files, sizes, n_images, pixels, pixels_on_device, row_pitch, image_stride);
}

int b200jpeg_decompress_batch_opts(b200jpeg_encoder *e, const b200jpeg_decompress_options *opts, const uint8_t *const *files,
                                   const size_t *sizes, int n_images, void *pixels, int pixels_on_device, size_t row_pitch, size_t image_stride)
{
  if (!e || !opts || !files || !sizes || !pixels || n_images <= 0) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  return decompress_rungs(e, Call{SINGLE_CALL, 1, n_images, opts, files, sizes}, View<void *>{&pixels, 0, 0}, View<size_t>{&row_pitch, 0, 0},
                          View<size_t>{&image_stride, 0, 0}, pixels_on_device);
}

int b200jpeg_decompress_yuv_batch(b200jpeg_encoder *e, const b200jpeg_decompress_options *opts, const uint8_t *const *files,
                                  const size_t *sizes, int n_images, uint8_t *const *planes, int planes_on_device,
                                  const size_t *plane_pitch, const size_t *plane_stride)
{
  return b200::decompress_yuv(e, opts, files, sizes, n_images, planes, planes_on_device, plane_pitch, plane_stride);
}

int b200jpeg_decode_yuv_batch(b200jpeg_encoder *e, const b200jpeg_params *p, const uint8_t *const *planes, int planes_on_device,
                              const size_t *plane_pitch, const size_t *plane_stride, void *pixels, int pixels_on_device,
                              size_t row_pitch, size_t image_stride, int n_images)
{
  return b200::decode_yuv(e, p, planes, planes_on_device, plane_pitch, plane_stride, pixels, pixels_on_device, row_pitch, image_stride, n_images);
}

int b200jpeg_recompress_batch(b200jpeg_encoder *e, const b200jpeg_params *p, const uint8_t *const *files, const size_t *sizes, int n_images)
{
  const b200jpeg_decompress_options o = b200jpeg_default_decompress_options();
  return b200jpeg_recompress_batch_opts(e, &o, p, files, sizes, n_images);
}

int b200jpeg_recompress_batch_opts(b200jpeg_encoder *e, const b200jpeg_decompress_options *opts, const b200jpeg_params *p,
                                   const uint8_t *const *files, const size_t *sizes, int n_images)
{
  if (!e || !opts || !p || !files || !sizes || n_images <= 0) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  return recompress_rungs(e, Call{SINGLE_CALL, 1, n_images, opts, files, sizes}, View<b200jpeg_params>{p, 0, 0});
}

int b200jpeg_decompress_renditions(b200jpeg_encoder *e, int n_renditions, const b200jpeg_decompress_options *opts, const uint8_t *const *files,
                                   const size_t *sizes, int n_images, void *const *pixels, int pixels_on_device,
                                   const size_t *row_pitch, const size_t *image_stride)
{
  if (e) e->files.clear();                       // a refused call leaves no outputs behind
  if (!e || n_renditions < 1 || !opts || !files || !sizes || n_images <= 0 || !pixels || !row_pitch || !image_stride) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  return decompress_rungs(e, Call{RENDITION_CALL, n_renditions, n_images, opts, files, sizes}, View<void *>{pixels, 1, 0}, View<size_t>{row_pitch, 1, 0},
                          View<size_t>{image_stride, 1, 0}, pixels_on_device);
}

int b200jpeg_decompress_mixed(b200jpeg_encoder *e, int n_renditions, const b200jpeg_decompress_options *opts, const uint8_t *const *files,
                              const size_t *sizes, int n_images, void *const *pixels, int pixels_on_device, const size_t *row_pitch)
{
  if (e) e->files.clear();
  if (!e || n_renditions < 1 || !opts || !files || !sizes || n_images <= 0 || !pixels || !row_pitch) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  if ((long long)n_renditions * n_images > INT_MAX) { set_error("%d renditions of %d images are more outputs than one call indexes", n_renditions, n_images); return B200JPEG_ERR_PARAM; }
  static const size_t none = 0;                  // each output is placed on its own: no image stride
  const size_t n = (size_t)n_images;
  return decompress_rungs(e, Call{MIXED_CALL, n_renditions, n_images, opts, files, sizes}, View<void *>{pixels, n, 1}, View<size_t>{row_pitch, n, 1},
                          View<size_t>{&none, 0, 0}, pixels_on_device);
}

int b200jpeg_recompress_mixed(b200jpeg_encoder *e, int n_renditions, const b200jpeg_decompress_options *opts, const b200jpeg_params *params,
                              const uint8_t *const *files, const size_t *sizes, int n_images)
{
  if (e) e->files.clear();
  if (!e || n_renditions < 1 || !opts || !params || !files || !sizes || n_images <= 0) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  if ((long long)n_renditions * n_images > INT_MAX) { set_error("%d renditions of %d images are more outputs than b200jpeg_get_output indexes", n_renditions, n_images); return B200JPEG_ERR_PARAM; }
  const int rc = recompress_rungs(e, Call{MIXED_CALL, n_renditions, n_images, opts, files, sizes}, View<b200jpeg_params>{params, (size_t)n_images, 1});
  if (rc && e) e->files.clear();
  return rc;
}

int b200jpeg_recompress_renditions(b200jpeg_encoder *e, int n_renditions, const b200jpeg_decompress_options *opts, const b200jpeg_params *params,
                                   const uint8_t *const *files, const size_t *sizes, int n_images)
{
  if (e) e->files.clear();
  if (!e || n_renditions < 1 || !opts || !params || !files || !sizes || n_images <= 0) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  if ((long long)n_renditions * n_images > INT_MAX) { set_error("%d renditions of %d images are more outputs than b200jpeg_get_output indexes", n_renditions, n_images); return B200JPEG_ERR_PARAM; }
  const int rc = recompress_rungs(e, Call{RENDITION_CALL, n_renditions, n_images, opts, files, sizes}, View<b200jpeg_params>{params, 1, 0});
  if (rc && e) e->files.clear();
  return rc;
}

int b200jpeg_decode_coefs_batch(b200jpeg_encoder *e, const uint8_t *const *files, const size_t *sizes, int n_images,
                                int16_t *const *planes, int planes_on_device, const size_t *row_pitch_blocks, const size_t *image_stride_blocks)
{
  if (!e || !planes || !row_pitch_blocks || !image_stride_blocks) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  e->dec.want_markers = false;
  int rc = decode_files(e, files, sizes, n_images);
  if (rc) return rc;
  const DecGeom &b = e->dec.geom[0];
  for (int c = 0; c < b.nc; c++) {
    const size_t wib = (size_t)b.wib[c], hib = (size_t)b.hib[c];
    if (!planes[c] || row_pitch_blocks[c] < wib || (n_images > 1 && image_stride_blocks[c] < row_pitch_blocks[c] * (hib - 1) + wib)) {
      set_error("coefficient plane %d: bad pointer, pitch or stride (needs %zu rows of %zu blocks)", c, hib, wib); return B200JPEG_ERR_PARAM;
    }
    const uint8_t *src = e->d_dec_planes.as<uint8_t>() + e->dec_plane_off[c];
    for (int i = 0; i < n_images; i++)
      CU(cudaMemcpy2DAsync(reinterpret_cast<uint8_t *>(planes[c]) + (size_t)i * image_stride_blocks[c] * 128, row_pitch_blocks[c] * 128,
                           src + (size_t)i * hib * wib * 128, wib * 128, wib * 128, hib, planes_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, e->stream));
  }
  CU(cudaStreamSynchronize(e->stream));
  e->pending_marks = 0;
  e->stage_names.clear(); e->stage_ms.clear(); e->stage_calls.clear();
  add_decode_stage_times(e);
  return B200JPEG_OK;
}

int b200jpeg_transcode_batch(b200jpeg_encoder *e, const b200jpeg_params *p, const uint8_t *const *files, const size_t *sizes, int n_images)
{
  return b200::transcode_files(e, p, nullptr, files, sizes, n_images);
}

int b200jpeg_transcode_batch_transform(b200jpeg_encoder *e, const b200jpeg_params *p, const b200jpeg_transform_info *t,
                                       const uint8_t *const *files, const size_t *sizes, int n_images)
{
  if (!t) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  return b200::transcode_files(e, p, t, files, sizes, n_images);
}

int b200jpeg_last_decode_sync(const b200jpeg_encoder *e, int *max_cta_rounds, long long *resync_subsequences)
{
  if (!e) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  if (max_cta_rounds) *max_cta_rounds = e->dec_rounds;
  if (resync_subsequences) *resync_subsequences = e->dec_redone;
  return B200JPEG_OK;
}

}  // extern "C"
