/*
 * tests/refdec.c -- TEST INFRASTRUCTURE (not product code).
 *
 * A driver around the UNMODIFIED reference library (oracle/_ref/libjpeg_ref.so): what rdjpeg.c, the JPEG input reader
 * of the reference's cjpeg, gets from it -- jpeg_read_header, jpeg_start_decompress and jpeg_read_scanlines on a
 * decompress object left at its defaults.  Built into build/librefdec.so where the reference build exists; the tests
 * and tools/make_golden.py --recompress compare the device decompression with it.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <setjmp.h>
#include <jpeglib.h>

struct my_err { struct jpeg_error_mgr pub; jmp_buf jb; };
static void my_exit(j_common_ptr c) { longjmp(((struct my_err *)c->err)->jb, 1); }
static void my_emit(j_common_ptr c, int lvl) { (void)c; (void)lvl; }

/* info: width, height, output_components, out_color_space, jpeg_color_space, warnings.  out (or NULL: header only)
 * receives height rows of width * output_components samples.  Returns 0, -1 for an error of the library, -2 when cap
 * is too small. */
int refdec_decompress(const unsigned char *jpeg, unsigned long size, unsigned char *out, unsigned long cap, int *info)
{
  struct jpeg_decompress_struct d;
  struct my_err err;
  d.err = jpeg_std_error(&err.pub);
  err.pub.error_exit = my_exit;
  err.pub.emit_message = my_emit;
  if (setjmp(err.jb)) { jpeg_destroy_decompress(&d); return -1; }
  jpeg_create_decompress(&d);
  jpeg_mem_src(&d, jpeg, size);
  jpeg_read_header(&d, TRUE);
  jpeg_start_decompress(&d);
  info[0] = (int)d.output_width; info[1] = (int)d.output_height; info[2] = d.output_components;
  info[3] = (int)d.out_color_space; info[4] = (int)d.jpeg_color_space;
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
