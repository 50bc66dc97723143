// The composite and per-node renders (composite_phases.h) and their reverse mode, one thread per ray.
#pragma once
#include "common.cuh"
#include "composite_phases.h"

namespace hold {

__global__ void __launch_bounds__(128) k_composite(CompositeArgs a) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= a.R) return;
  composite_ray(a, r);
}

__global__ void __launch_bounds__(128) k_composite_bwd(CompositeBwdArgs a) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= a.R) return;
  composite_bwd_ray(a, r);
}

}  // namespace hold
