// internal.h -- shared declarations inside libb200jpeg (not installed).
#pragma once
#include "b200jpeg.h"
namespace b200 {
void set_error(const char *fmt, ...);
// lossless mode as the reference's validate_script detects it (jcmaster.c:302-311): the script's first entry has
// Ss != 0 and Se == 0 (the scan search skips the check, jcmaster.c:285-291)
bool is_lossless(const b200jpeg_params *p);
// the parameter block jpeg_start_compress works with in lossless mode (jcmaster.c:1072-1094): default colour space,
// 1x1 sampling, no smoothing, optimal tables; b200jpeg_enable_lossless's one-scan script follows the new component count
void lossless_start(const b200jpeg_params *in, b200jpeg_params *out);
}
