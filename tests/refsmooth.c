/*
 * tests/refsmooth.c -- TEST INFRASTRUCTURE (not product code).
 *
 * A driver around the UNMODIFIED reference library (oracle/_ref/libjpeg_ref.so): jpeg_read_header,
 * jpeg_start_decompress and jpeg_read_scanlines on a decompress object at its defaults except do_block_smoothing,
 * which the caller sets.  tools/make_golden.py --progressive decodes each progressive source with smoothing on and off:
 * where the pixels differ, the reference block-smooths the file.  Built into build/librefsmooth.so where the reference
 * build exists.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <setjmp.h>
#include <jpeglib.h>

struct my_err { struct jpeg_error_mgr pub; jmp_buf jb; };
static void my_exit(j_common_ptr c) { longjmp(((struct my_err *)c->err)->jb, 1); }
static void my_emit(j_common_ptr c, int lvl) { (void)c; (void)lvl; }

/* out receives output_height rows of output_width * output_components samples (cap bytes at most).  Returns the
 * number of bytes written, -1 for an error of the library, -2 when cap is too small. */
long refsmooth_decompress(const unsigned char *jpeg, unsigned long size, int smoothing, unsigned char *out, unsigned long cap)
{
  struct jpeg_decompress_struct d;
  struct my_err err;
  unsigned long row;
  d.err = jpeg_std_error(&err.pub);
  err.pub.error_exit = my_exit;
  err.pub.emit_message = my_emit;
  if (setjmp(err.jb)) { jpeg_destroy_decompress(&d); return -1; }
  jpeg_create_decompress(&d);
  jpeg_mem_src(&d, jpeg, size);
  jpeg_read_header(&d, TRUE);
  d.do_block_smoothing = smoothing ? TRUE : FALSE;
  jpeg_start_decompress(&d);
  row = (unsigned long)d.output_width * d.output_components;
  if (cap < row * d.output_height) { jpeg_destroy_decompress(&d); return -2; }
  while (d.output_scanline < d.output_height) {
    JSAMPROW r = out + row * d.output_scanline;
    jpeg_read_scanlines(&d, &r, 1);
  }
  jpeg_finish_decompress(&d);
  jpeg_destroy_decompress(&d);
  return (long)(row * d.output_height);
}
