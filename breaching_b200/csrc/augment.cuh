// Candidate augmentations (augment.cu): plan of the linear view pipeline and the per-iteration random draws.
#pragma once
#include "common.cuh"

namespace bre {

constexpr int AUG_MAX_STEPS = 4;     // permutation steps (discrete_shift / flip) in config order
constexpr int AUG_MAX_BATCH = 64;    // per-image uniforms of the continuous shift
constexpr int AUG_MAX_STAGES = 8;    // stages of the view pipeline (see AugStage)
constexpr int AUG_CS_MAX_SIDE = 1024; // continuous_shift: the per-image tap tables of both axes fit 48 KB of shared memory
enum AugKind { AUG_SHIFT = 1, AUG_FLIP = 2 };
// continuous_shift sampling (grid_sample mode / padding_mode; "circular" is a zeros-padded wrap of the grid, cs_circular)
enum AugCsMode { AUG_CS_BILINEAR = 0, AUG_CS_NEAREST = 1, AUG_CS_BICUBIC = 2 };
enum AugCsPadding { AUG_CS_ZEROS = 0, AUG_CS_BORDER = 1, AUG_CS_REFLECTION = 2 };
// A stage of the view pipeline.  PIXEL: a maximal run of the shape-keeping kinds (discrete_shift, flip, continuous_shift,
// colorjitter) on the fused kernels below, described by its AugPlan.  RESAMPLE: a window of the input resized bilinearly
// (zoom, centerzoom, focus).  BLUR: the binomial depthwise convolution of antialias.
enum AugStageKind { AUG_STAGE_PIXEL = 0, AUG_STAGE_RESAMPLE = 1, AUG_STAGE_BLUR = 2 };

struct AugPlan {
  int n_steps;
  int kind[AUG_MAX_STEPS];
  float p0[AUG_MAX_STEPS];           // discrete_shift: lim ; flip: p
  int cs_enabled, cs_circular;       // continuous_shift (applied after the permutation steps)
  float cs_shift;
  const float* cj_scale;             // colour affine per (n, c): out = in * scale + shift (composite of all colorjitter steps), may be null
  const float* cj_shift;
  unsigned long long seed;
  int cs_mode, cs_padding;           // AugCsMode, AugCsPadding
  int cs_fliplr, cs_flipud;          // grid flips: each image negates its x (y) coordinate when its third (fourth) uniform is > 0.5
};
struct AugDraws {
  int o1[AUG_MAX_STEPS], o2[AUG_MAX_STEPS];   // discrete_shift: the two roll offsets ; flip: o1 = flipped? ; focus: o1[0], o2[0] = window corner
  float sx[AUG_MAX_BATCH], sy[AUG_MAX_BATCH]; // continuous_shift: uniforms in [0, 1) per image (randgen[:, 0], randgen[:, 1])
  int flr[AUG_MAX_BATCH], fud[AUG_MAX_BATCH]; // continuous_shift: 1 = this image's grid is flipped left-right / up-down
};
struct AugStage {
  int kind;                          // AugStageKind
  int C, Hi, Wi, Ho, Wo;             // input and output plane shape (the batch is the candidate's)
  int y0, x0, wh, ww;                // RESAMPLE: window corner and size (corner drawn per forward when focus != 0)
  int focus;                         // RESAMPLE: Focus, corner = clamp(trunc(pert + in // 2 - size // 2)), pert uniform in [-std, std)
  float focus_std;
  int width, stride;                 // BLUR: binomial width (1..7), stride; zero padding width // 2
};
// all stages of one pipeline: the draw kernel takes it by value (one launch draws every stage)
struct AugPipeline {
  int n_stages;
  unsigned long long seed;           // focus corners: Philox(seed, iteration, stage); PIXEL stages draw with their plan's seed
  AugStage st[AUG_MAX_STAGES];
  AugPlan plan[AUG_MAX_STAGES];      // PIXEL stages only
};

// F.interpolate(mode="bilinear", align_corners=False) along one axis: output index o of `out` samples the input of extent `in`
// at (o + 0.5) * scale - 0.5 (scale = in / out), clamped at 0; neighbours i0 = floor and i1 = min(i0 + 1, in - 1) with weights
// (1 - l, l).  At the last index both weights land on in - 1.  Shared by the multi-scale resize and the RESAMPLE stage.
__device__ __forceinline__ void bilinear_src(int o, float scale, int in, int& i0, int& i1, float& l) {
  float f = ((float)o + 0.5f) * scale - 0.5f;
  f = f < 0.f ? 0.f : f;
  i0 = (int)f;
  i1 = i0 + (i0 < in - 1 ? 1 : 0);
  l = f - (float)i0;
}

// the draws of every stage of this iteration -> draws[stage]
int launch_aug_draws(const AugPipeline& pipe, const Scalars* sc, AugDraws* draws, int N, cudaStream_t s);
int launch_aug_view(const float* x, float* out, int N, int C, int H, int W, const AugPlan& plan, const AugDraws* draws, cudaStream_t s);
int launch_aug_pull(float* g, float* tmp, float* gx, int N, int C, int H, int W, const AugPlan& plan, const AugDraws* draws, cudaStream_t s);
// RESAMPLE / BLUR: view x [N, C, Hi, Wi] -> out [N, C, Ho, Wo]; pull g [N, C, Ho, Wo] -> gx [N, C, Hi, Wi] (fixed-order gathers;
// the RESAMPLE pull-back is separable and needs tmp of N * C * Ho * ww floats)
int launch_aug_resample(const float* x, float* out, int N, const AugStage& st, const AugDraws* draws, bool transpose, float* tmp, cudaStream_t s);
int launch_aug_blur(const float* x, float* out, int N, const AugStage& st, bool transpose, cudaStream_t s);

}  // namespace bre
