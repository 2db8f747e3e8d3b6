// transform.cpp -- host parameter logic of jpegtran's lossless transforms (transupp.c as built with
// JPEG_LIB_VERSION 62: DCT blocks of 8x8, no scaling).  The coefficient import (k_import_coefs) applies the block
// mapping filled in here.
#include "b200jpeg.h"
#include "internal.h"

#include <algorithm>

using b200::set_error;

namespace {

bool transposes(int x)
{
  return x == B200JPEG_XFORM_TRANSPOSE || x == B200JPEG_XFORM_TRANSVERSE || x == B200JPEG_XFORM_ROT_90 || x == B200JPEG_XFORM_ROT_270;
}

// jtransform_perfect_transform (transupp.c:2273-2303)
bool perfect(unsigned w, unsigned h, unsigned mw, unsigned mh, int x)
{
  switch (x) {
  case B200JPEG_XFORM_FLIP_H: case B200JPEG_XFORM_ROT_270: return w % mw == 0;
  case B200JPEG_XFORM_FLIP_V: case B200JPEG_XFORM_ROT_90: return h % mh == 0;
  case B200JPEG_XFORM_TRANSVERSE: case B200JPEG_XFORM_ROT_180: return w % mw == 0 && h % mh == 0;
  default: return true;
  }
}

// the crop checks of jtransform_request_workspace (transupp.c:1591-1628) along one axis; -1: JERR_BAD_CROP_SPEC,
// 1: crop extension (the region is larger than the image), 0: a plain crop.  `size` receives the region's extent.
int crop_axis(int size_set, unsigned size, unsigned off, unsigned full, int transform, unsigned &out)
{
  if (size_set == B200JPEG_CROP_UNSET) {
    if (off >= full) return -1;
    out = full - off;
    return 0;
  }
  out = size;
  if (size > full) return (transform != B200JPEG_XFORM_NONE || off >= size || off > size - full) ? -1 : 1;
  return (off >= full || size == 0 || off > full - size) ? -1 : 0;
}

int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }

}  // namespace

extern "C" int b200jpeg_transform_setup(const b200jpeg_source_info *src, b200jpeg_transform_info *t, b200jpeg_params *p)
{
  if (!src || !t || !p) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  const int xf = t->transform;
  if (xf < B200JPEG_XFORM_NONE || xf > B200JPEG_XFORM_ROT_270) { set_error("unknown transform %d", xf); return B200JPEG_ERR_PARAM; }
  const int kinds[4] = {t->crop_width_set, t->crop_height_set, t->crop_xoffset_set, t->crop_yoffset_set};
  for (int k : kinds)
    if (k < B200JPEG_CROP_UNSET || k > B200JPEG_CROP_REFLECT) { set_error("unknown crop kind %d", k); return B200JPEG_ERR_PARAM; }
  const int snc = src->num_components;
  if (snc < 1 || snc > B200JPEG_MAX_COMPONENTS || p->num_components != snc) { set_error("the parameter block has %d components, the source %d", p->num_components, snc); return B200JPEG_ERR_PARAM; }
  int hmax = 1, vmax = 1;
  for (int ci = 0; ci < snc; ci++) { hmax = std::max(hmax, src->h_samp_factor[ci]); vmax = std::max(vmax, src->v_samp_factor[ci]); }
  const unsigned W = (unsigned)src->image_width, H = (unsigned)src->image_height;
  const bool T = transposes(xf);

  // jtransform_request_workspace (transupp.c:1495-1826)
  const int nc = (t->force_grayscale && src->jpeg_color_space == B200JPEG_CS_YCbCr && snc == 3) ? 1 : snc;
  const unsigned mw = nc == 1 ? 8u : (unsigned)hmax * 8, mh = nc == 1 ? 8u : (unsigned)vmax * 8;
  if (t->perfect && !perfect(W, H, mw, mh, xf)) { set_error("transformation is not perfect"); return B200JPEG_ERR_PARAM; }
  unsigned ow = T ? H : W, oh = T ? W : H;
  const unsigned iw = T ? mh : mw, ih = T ? mw : mh;
  unsigned xoff = 0, yoff = 0;
  if (t->crop) {
    const unsigned cx = t->crop_xoffset_set == B200JPEG_CROP_UNSET ? 0 : t->crop_xoffset;
    const unsigned cy = t->crop_yoffset_set == B200JPEG_CROP_UNSET ? 0 : t->crop_yoffset;
    unsigned cw = 0, ch = 0;
    const int ew = crop_axis(t->crop_width_set, t->crop_width, cx, ow, xf, cw);
    if (ew < 0) { set_error("Invalid crop request"); return B200JPEG_ERR_PARAM; }
    const int eh = crop_axis(t->crop_height_set, t->crop_height, cy, oh, xf, ch);
    if (eh < 0) { set_error("Invalid crop request"); return B200JPEG_ERR_PARAM; }
    if (ew > 0 || eh > 0) { set_error("crop extension (a crop region of %ux%u on a %ux%u image, do_crop_ext_*) is not on the device path", cw, ch, ow, oh); return B200JPEG_ERR_UNSUPPORTED; }
    const unsigned xo = t->crop_xoffset_set != B200JPEG_CROP_NEG ? cx : ow - cw - cx;
    const unsigned yo = t->crop_yoffset_set != B200JPEG_CROP_NEG ? cy : oh - ch - cy;
    ow = t->crop_width_set == B200JPEG_CROP_FORCE ? cw : cw + xo % iw;
    oh = t->crop_height_set == B200JPEG_CROP_FORCE ? ch : ch + yo % ih;
    xoff = xo / iw; yoff = yo / ih;
  }
  // trim_right_edge / trim_bottom_edge (transupp.c:1455-1475) against the source extent along that destination axis
  auto trim_right = [&](unsigned full) { const unsigned c = ow / iw; if (c > 0 && xoff + c == full / iw) ow = c * iw; };
  auto trim_bottom = [&](unsigned full) { const unsigned r = oh / ih; if (r > 0 && yoff + r == full / ih) oh = r * ih; };
  if (t->trim) {
    switch (xf) {
    case B200JPEG_XFORM_FLIP_H: trim_right(W); break;
    case B200JPEG_XFORM_FLIP_V: trim_bottom(H); break;
    case B200JPEG_XFORM_TRANSVERSE: trim_right(H); trim_bottom(W); break;
    case B200JPEG_XFORM_ROT_90: trim_right(H); break;
    case B200JPEG_XFORM_ROT_180: trim_right(W); trim_bottom(H); break;
    case B200JPEG_XFORM_ROT_270: trim_bottom(W); break;
    default: break;
    }
  }

  // jtransform_adjust_parameters (transupp.c:2042-2113)
  b200jpeg_params q = *p;
  if (t->force_grayscale) {
    const bool ok = ((q.jpeg_color_space == B200JPEG_CS_YCbCr && q.num_components == 3) || (q.jpeg_color_space == B200JPEG_CS_GRAYSCALE && q.num_components == 1)) &&
                    src->h_samp_factor[0] == hmax && src->v_samp_factor[0] == vmax;
    if (!ok) { set_error("Unsupported color conversion request"); return B200JPEG_ERR_PARAM; }
    const int tq = q.comp_info[0].quant_tbl_no;
    const int rc = b200jpeg_set_colorspace(&q, B200JPEG_CS_GRAYSCALE);
    if (rc) return rc;
    q.comp_info[0].quant_tbl_no = tq;
  } else if (nc == 1) {
    q.comp_info[0].h_samp_factor = q.comp_info[0].v_samp_factor = 1;
  }
  q.image_width = (int)ow; q.image_height = (int)oh;
  if (T) {                                            // transpose_critical_parameters (transupp.c:1831-1872)
    for (int ci = 0; ci < q.num_components; ci++) std::swap(q.comp_info[ci].h_samp_factor, q.comp_info[ci].v_samp_factor);
    for (int s = 0; s < B200JPEG_NUM_QUANT_TBLS; s++)
      if (q.quant_tbl_present[s])
        for (int i = 0; i < 8; i++)
          for (int j = 0; j < i; j++) std::swap(q.quant_tbl[s][i * 8 + j], q.quant_tbl[s][j * 8 + i]);
  }

  // the block mapping of the do_* routines (transupp.c:727-1357): the mirrorable extent of each destination axis is
  // the source's whole iMCUs along it, in the destination's blocks
  int dh = 1, dv = 1;
  for (int ci = 0; ci < q.num_components; ci++) { dh = std::max(dh, q.comp_info[ci].h_samp_factor); dv = std::max(dv, q.comp_info[ci].v_samp_factor); }
  const unsigned src_x = T ? H : W, src_y = T ? W : H;   // source extent along the destination's x / y axis
  const bool mx = xf == B200JPEG_XFORM_FLIP_H || xf == B200JPEG_XFORM_TRANSVERSE || xf == B200JPEG_XFORM_ROT_90 || xf == B200JPEG_XFORM_ROT_180;
  const bool my = xf == B200JPEG_XFORM_FLIP_V || xf == B200JPEG_XFORM_TRANSVERSE || xf == B200JPEG_XFORM_ROT_270 || xf == B200JPEG_XFORM_ROT_180;
  b200jpeg_transform_info r = *t;
  r.transposed = T;
  for (int ci = 0; ci < B200JPEG_MAX_COMPONENTS; ci++) {
    r.x_crop_blocks[ci] = r.y_crop_blocks[ci] = r.x_mirror[ci] = r.y_mirror[ci] = r.src_wib[ci] = r.src_hib[ci] = 0;
    if (ci >= q.num_components) continue;
    const int h = q.comp_info[ci].h_samp_factor, v = q.comp_info[ci].v_samp_factor;
    r.x_crop_blocks[ci] = (int)xoff * h; r.y_crop_blocks[ci] = (int)yoff * v;
    r.x_mirror[ci] = mx ? (int)(src_x / ((unsigned)dh * 8)) * h : 0;
    r.y_mirror[ci] = my ? (int)(src_y / ((unsigned)dv * 8)) * v : 0;
    r.src_wib[ci] = ceil_div((long long)W * src->h_samp_factor[ci], (long long)hmax * 8);
    r.src_hib[ci] = ceil_div((long long)H * src->v_samp_factor[ci], (long long)vmax * 8);
    // every real destination block must read a real source block (the source planes hold no iMCU padding)
    const int dwib = ceil_div((long long)ow * h, (long long)dh * 8), dhib = ceil_div((long long)oh * v, (long long)dv * 8);
    const int lim_x = T ? r.src_hib[ci] : r.src_wib[ci], lim_y = T ? r.src_wib[ci] : r.src_hib[ci];
    for (int pass = 0; pass < 2; pass++) {
      const int n = pass ? dhib : dwib, cb = pass ? r.y_crop_blocks[ci] : r.x_crop_blocks[ci];
      const int m = pass ? r.y_mirror[ci] : r.x_mirror[ci], lim = pass ? lim_y : lim_x;
      for (int d = 0; d < n; d++) {
        int a = d + cb;
        if (a < m) a = m - 1 - a;
        if (a < 0 || a >= lim) {
          set_error("transform %d: destination component %d %s %d would read source block %d of %d (iMCU padding)", xf, ci, pass ? "row" : "column", d, a, lim);
          return B200JPEG_ERR_UNSUPPORTED;
        }
      }
    }
  }
  r.num_components = q.num_components;
  r.output_width = (int)ow; r.output_height = (int)oh;
  r.iMCU_sample_width = (int)iw; r.iMCU_sample_height = (int)ih;
  r.x_crop_offset = (int)xoff; r.y_crop_offset = (int)yoff;
  *t = r; *p = q;
  return B200JPEG_OK;
}
