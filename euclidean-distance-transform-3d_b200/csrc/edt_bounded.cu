// The bounded transforms' window and cut kernels for every label width (see edt_bounded.cuh).
#include "edt_bounded.cuh"
EDT_INSTANTIATE_BOUNDED(1)
EDT_INSTANTIATE_BOUNDED(2)
EDT_INSTANTIATE_BOUNDED(4)
EDT_INSTANTIATE_BOUNDED(8)
