// The parabolic erosion and dilation passes (see edt_parabolic.cuh).
#include "edt_parabolic.cuh"
