/*
 * tests/refdecopt.c -- TEST INFRASTRUCTURE (not product code).
 *
 * A driver around the UNMODIFIED reference library (oracle/_ref/libjpeg_ref.so): jpeg_read_header, then the
 * decompress options djpeg sets (scale_num / scale_denom, dct_method, do_fancy_upsampling, out_color_space; -1 keeps
 * default_decompress_parms' choice), jpeg_start_decompress and jpeg_read_scanlines.  Built into
 * build/librefdecopt.so where the reference build exists; tests/test_decompress_options.py and
 * tools/make_golden.py --decompress-options compare the device decompression with it.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <setjmp.h>
#include <jpeglib.h>

struct my_err { struct jpeg_error_mgr pub; jmp_buf jb; };
static void my_exit(j_common_ptr c) { longjmp(((struct my_err *)c->err)->jb, 1); }
static void my_emit(j_common_ptr c, int lvl) { (void)c; (void)lvl; }

/* opts: scale_num, scale_denom, dct_method, do_fancy_upsampling, out_color_space (-1: default).
 * info (at least 20 ints): output_width, output_height, output_components, out_color_space, jpeg_color_space,
 * warnings, num_components, then per component (up to 4) DCT_scaled_size, downsampled_width, downsampled_height.
 * out (or NULL: jpeg_start_decompress only) receives output_height rows of output_width * output_components samples.
 * msg (or NULL) receives the library's message when it fails.  Returns 0, -1 for an error of the library, -2 when
 * cap is too small. */
int refdecopt_decompress(const unsigned char *jpeg, unsigned long size, const int *opts, unsigned char *out, unsigned long cap, int *info, char *msg)
{
  struct jpeg_decompress_struct d;
  struct my_err err;
  int ci;
  d.err = jpeg_std_error(&err.pub);
  err.pub.error_exit = my_exit;
  err.pub.emit_message = my_emit;
  if (setjmp(err.jb)) {
    if (msg) (*err.pub.format_message)((j_common_ptr)&d, msg);
    jpeg_destroy_decompress(&d);
    return -1;
  }
  jpeg_create_decompress(&d);
  jpeg_mem_src(&d, jpeg, size);
  jpeg_read_header(&d, TRUE);
  d.scale_num = (unsigned)opts[0];
  d.scale_denom = (unsigned)opts[1];
  d.dct_method = (J_DCT_METHOD)opts[2];
  d.do_fancy_upsampling = opts[3] ? TRUE : FALSE;
  if (opts[4] >= 0) d.out_color_space = (J_COLOR_SPACE)opts[4];
  jpeg_start_decompress(&d);
  info[0] = (int)d.output_width; info[1] = (int)d.output_height; info[2] = d.output_components;
  info[3] = (int)d.out_color_space; info[4] = (int)d.jpeg_color_space; info[6] = d.num_components;
  for (ci = 0; ci < d.num_components && ci < 4; ci++) {
    info[7 + 3 * ci] = d.comp_info[ci].DCT_scaled_size;
    info[8 + 3 * ci] = (int)d.comp_info[ci].downsampled_width;
    info[9 + 3 * ci] = (int)d.comp_info[ci].downsampled_height;
  }
  if (out) {
    const unsigned long row = (unsigned long)d.output_width * d.output_components;
    if (cap < row * d.output_height) { jpeg_destroy_decompress(&d); return -2; }
    while (d.output_scanline < d.output_height) {
      JSAMPROW r = out + row * d.output_scanline;
      jpeg_read_scanlines(&d, &r, 1);
    }
    jpeg_finish_decompress(&d);
  }
  info[5] = (int)err.pub.num_warnings;
  jpeg_destroy_decompress(&d);
  return 0;
}
