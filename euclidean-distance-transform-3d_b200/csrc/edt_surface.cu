// The surface-distance kernels for every label width (see edt_surface.cuh).
#include "edt_surface.cuh"
EDT_INSTANTIATE_SURFACE(1)
EDT_INSTANTIATE_SURFACE(2)
EDT_INSTANTIATE_SURFACE(4)
EDT_INSTANTIATE_SURFACE(8)
