// Diffuse-only instantiation of the render kernels: the lean kernels (rb_kernels_lean.cu) compiled once more with RB_DIFFUSE, i.e.
// with "no material computes specular lighting, uses vertex colours or has a normal map" as compile-time facts as well, inside
// namespace rb_diffuse.  rb_render launches these (rb_diffuse::render_kernels()) when the scene qualifies for the lean kernels and
// every material is of this kind, the material of most shape and pose optimisations.  Measured on C2: see DESIGN.md section 6.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <string>
#include <vector>

#include "../../include/redner_b200.h"
#include "rb_kernel_set.h"

#define RB_LEAN 1
#define RB_DIFFUSE 1
namespace rb_diffuse {
#include "rb_render.cuh"
#include "rb_kernels_body.cuh"
} // namespace rb_diffuse
