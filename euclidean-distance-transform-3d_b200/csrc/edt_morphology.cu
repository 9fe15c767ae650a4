// The spherical morphology's stores for every label width (see edt_morphology.cuh): the window pass
// that writes a label or mask, the select after an unbounded last pass, and the fold of float labels.
#include "edt_morphology.cuh"
