// decode_list.cu -- the decoders' stream-list instantiations (a mixed byte session's launches over the streams of one
// answer type), built from decode_formats.cu in a translation unit of their own: every kernel of decode_formats.cu
// then compiles to the same code whether or not these exist.
#define RPL_DECODE_LIST
#include "decode_formats.cu"
