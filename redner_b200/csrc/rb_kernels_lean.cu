// Feature-free instantiation of the render kernels: the very same source (rb_kernels_body.cuh and every per-sample header)
// compiled with RB_LEAN, i.e. with "no environment map, pinhole camera without lens model, channels == [radiance]" as
// compile-time facts, inside namespace rb_lean.  rb_render launches these (rb_lean::render_kernels()) when the scene and the
// options allow it; the general kernels in rb_kernels.cu cover everything else.  Measured on C2: see DESIGN.md section 6.
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
namespace rb_lean {
#include "rb_render.cuh"
#include "rb_kernels_body.cuh"
} // namespace rb_lean
