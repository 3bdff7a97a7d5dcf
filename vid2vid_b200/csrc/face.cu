// Kernels of the edge2face first-frame generator that are not convolutions (models/vid2vid_model_G.py:231-320):
//   instance_mean   Encoder.forward's instance-wise average pooling (models/networks.py:617-632): every value of channel c
//                   of image n becomes the mean of that channel over the pixels of image n that share its id.  One block
//                   per (n, c) plane; the ids are taken in groups of 8 held in registers, each thread adds its fixed pixels
//                   in double, and the block reduces in a fixed order (no float atomics: the same inputs give the same bits
//                   on every run and every graph replay).  The mean is divided once in double and rounded to fp32.
//   face_features   get_face_features (models/vid2vid_model_G.py:290-320) + dists_min (models/base_model.py:136-144): the
//                   pooled feature at the first pixel of each label present (integer atomicMin of the flat (n, y, x)
//                   index), squared distances to the rows of the packed features table in double, the first minimum, and
//                   the chosen rows painted over the part map.  The search runs once per group of images: the whole batch
//                   (the reference's get_face_features) or each image on its own (B independent clips, one block each).
#include <climits>

#include "../../include/v2v_b200.h"
#include "v2v_internal.h"

namespace v2v {

void set_error(const char* fmt, ...);

constexpr int FACE_MAX_LABELS = V2V_FACE_MAX_LABELS, FACE_MAX_FEAT = V2V_FACE_MAX_FEAT;
enum { FACE_ERR_ID = 1, FACE_ERR_ROWS = 2 };

__device__ __forceinline__ bool valid_id(float v, int n_ids) {
  return v >= 0.f && v < (float)n_ids && v == floorf(v);
}

// ------------------------------------------------------------------------------ instance mean
constexpr int IM_THREADS = 1024, IM_GROUP = 8;

__device__ __forceinline__ double warp_sum_dbl(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ long long warp_sum_ll(long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Pixels with an invalid id set FACE_ERR_ID in *err and are written as NaN (they belong to no instance).
__global__ void __launch_bounds__(IM_THREADS) instance_mean_kernel(const float* __restrict__ x, const float* __restrict__ inst,
                                                                   float* out, int C, int HW, int n_ids, int* err) {
  const int plane = blockIdx.x, n = plane / C;
  const float* xp = x + (size_t)plane * HW;
  const float* ip = inst + (size_t)n * HW;
  float* op = out + (size_t)plane * HW;
  __shared__ double s_sum[IM_THREADS / 32][IM_GROUP];
  __shared__ long long s_cnt[IM_THREADS / 32][IM_GROUP];
  __shared__ float s_mean[IM_GROUP];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int k0 = 0; k0 < n_ids; k0 += IM_GROUP) {
    double sum[IM_GROUP];
    long long cnt[IM_GROUP];
#pragma unroll
    for (int j = 0; j < IM_GROUP; ++j) { sum[j] = 0.0; cnt[j] = 0; }
    for (int p = threadIdx.x; p < HW; p += IM_THREADS) {
      const float id = __ldg(ip + p);
      if (k0 == 0 && !valid_id(id, n_ids)) { atomicOr(err, FACE_ERR_ID); continue; }
      const int k = (int)id - k0;
      if (k < 0 || k >= IM_GROUP) continue;
      const double v = (double)xp[p];
#pragma unroll
      for (int j = 0; j < IM_GROUP; ++j)
        if (j == k) { sum[j] += v; ++cnt[j]; }
    }
#pragma unroll
    for (int j = 0; j < IM_GROUP; ++j) {
      const double s = warp_sum_dbl(sum[j]);
      const long long c = warp_sum_ll(cnt[j]);
      if (lane == 0) { s_sum[warp][j] = s; s_cnt[warp][j] = c; }
    }
    __syncthreads();
    if (threadIdx.x < IM_GROUP) {
      double s = 0.0;
      long long c = 0;
      for (int w = 0; w < IM_THREADS / 32; ++w) { s += s_sum[w][threadIdx.x]; c += s_cnt[w][threadIdx.x]; }
      s_mean[threadIdx.x] = c ? (float)(s / (double)c) : 0.f;
    }
    __syncthreads();
    // every pixel of this group's ids is rewritten only after all of them were read (out may alias x)
    for (int p = threadIdx.x; p < HW; p += IM_THREADS) {
      const float id = __ldg(ip + p);
      if (!valid_id(id, n_ids)) { if (k0 == 0) op[p] = __int_as_float(0x7fc00000); continue; }
      const int k = (int)id - k0;
      if (k >= 0 && k < IM_GROUP) op[p] = s_mean[k];
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------ face features
struct FaceFeatParams {
  const float* pooled;     // (N, feat_num, H, W)
  const float* inst;       // (N, 1, H, W) label ids
  const float* table;      // (n_labels, max_rows, stride)
  float* out;              // (N, feat_num, H, W)
  int* chosen;             // device int32 [groups]
  int* first;              // scratch [groups][FACE_MAX_LABELS]: first flat (n, y, x) index of each label, >= N * H * W = absent
  int* bad;                // scratch [groups]: the group's part map holds an invalid id
  int* err;
  int rows[FACE_MAX_LABELS];
  int n_labels, max_rows, num_images, feat_num, stride, N, H, W;
  int per_image;           // 0: one group (the whole batch); 1: one group per image
  __device__ int group_of(int n) const { return per_image ? n : 0; }
};

__global__ void __launch_bounds__(256) face_first_index_kernel(FaceFeatParams p) {
  const int total = p.N * p.H * p.W;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const float id = __ldg(p.inst + i);
    const int g = p.group_of(i / (p.H * p.W));
    if (!valid_id(id, p.n_labels)) { atomicOr(p.err, FACE_ERR_ID); atomicOr(p.bad + g, 1); continue; }
    atomicMin(p.first + g * FACE_MAX_LABELS + (int)id, i);
  }
}

// One block per group.  dists[m] = sum_k sum_label (feat_ori[label][k] - table[label][m][k])^2 over the labels present, in double, in
// the reference's order (labels first, then k); the first minimum over m < num_images wins.
__global__ void __launch_bounds__(256) face_choose_kernel(FaceFeatParams p) {
  __shared__ float s_ori[FACE_MAX_LABELS][FACE_MAX_FEAT];
  __shared__ int s_present[FACE_MAX_LABELS];
  __shared__ double s_d[256];
  __shared__ int s_m[256];
  const int HW = p.H * p.W, g = blockIdx.x;
  bool bad = false;
  for (int l = 0; l < p.n_labels; ++l) {
    const int f = p.first[g * FACE_MAX_LABELS + l];
    const bool present = f < p.N * HW;
    if (threadIdx.x == 0) s_present[l] = present;
    if (present && p.rows[l] < p.num_images) bad = true;
    if (present) {
      const int n = f / HW, px = f - n * HW;
      for (int k = threadIdx.x; k < p.feat_num; k += blockDim.x) s_ori[l][k] = p.pooled[((size_t)n * p.feat_num + k) * HW + px];
    }
  }
  if (bad || p.bad[g]) {
    if (threadIdx.x == 0) { if (bad) atomicOr(p.err, FACE_ERR_ROWS); p.chosen[g] = -1; }
    return;
  }
  __syncthreads();
  double best = INFINITY;
  int best_m = INT_MAX;
  for (int m = threadIdx.x; m < p.num_images; m += blockDim.x) {        // increasing m: strict < keeps the first minimum
    double d = 0.0;
    for (int k = 0; k < p.feat_num; ++k) {
      double dk = 0.0;
      for (int l = 0; l < p.n_labels; ++l) {
        if (!s_present[l]) continue;                                      // absent labels contribute nothing
        const double e = (double)s_ori[l][k] - (double)__ldg(p.table + ((size_t)l * p.max_rows + m) * p.stride + k);
        dk += e * e;
      }
      d += dk;
    }
    if (d < best) { best = d; best_m = m; }
  }
  s_d[threadIdx.x] = best; s_m[threadIdx.x] = best_m;
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      const double d2 = s_d[threadIdx.x + o];
      const int m2 = s_m[threadIdx.x + o];
      if (d2 < s_d[threadIdx.x] || (d2 == s_d[threadIdx.x] && m2 < s_m[threadIdx.x])) { s_d[threadIdx.x] = d2; s_m[threadIdx.x] = m2; }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) p.chosen[g] = s_m[0] == INT_MAX ? 0 : s_m[0];
}

// out[n, k, y, x] = table[label][min(chosen, rows[label] - 1)][k] with the chosen index of image n's group; NaN when no
// index was chosen (an error was flagged)
__global__ void __launch_bounds__(256) face_paint_kernel(FaceFeatParams p) {
  const int HW = p.H * p.W;
  const size_t total = (size_t)p.N * p.feat_num * HW;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int px = (int)(i % HW);
    const size_t t = i / HW;
    const int k = (int)(t % p.feat_num), n = (int)(t / p.feat_num);
    const float id = __ldg(p.inst + (size_t)n * HW + px);
    const int chosen = p.chosen[p.group_of(n)];
    float v = __int_as_float(0x7fc00000);
    if (chosen >= 0 && valid_id(id, p.n_labels)) {
      const int l = (int)id;
      v = __ldg(p.table + ((size_t)l * p.max_rows + min(chosen, p.rows[l] - 1)) * p.stride + k);
    }
    p.out[i] = v;
  }
}

static int grid_of(size_t total) {
  const size_t b = (total + 255) / 256, cap = (size_t)device_sm_count() * 8;
  return (int)(b < cap ? (b ? b : 1) : cap);
}

#define FACE_CUDA(expr)                                                        \
  do {                                                                         \
    cudaError_t e__ = (expr);                                                  \
    if (e__ != cudaSuccess) {                                                  \
      set_error("%s failed: %s", #expr, cudaGetErrorString(e__));              \
      return (int)e__;                                                         \
    }                                                                          \
  } while (0)
#define FACE_REQUIRE(cond, ...)    \
  do {                             \
    if (!(cond)) {                 \
      set_error(__VA_ARGS__);      \
      return V2V_ERR_INVALID;      \
    }                              \
  } while (0)

// Scratch ints on the stream (stream-ordered allocation, so the ops stay capturable into a CUDA graph).  Outside capture the
// error flag is read back after the kernels and turned into an error code; inside capture the host cannot wait, and the
// flagged outputs are NaN (instance_mean) or chosen = -1 with a NaN feature map (face_features).
struct Scratch {
  int* p = nullptr;
  cudaStream_t s;
  explicit Scratch(cudaStream_t s_) : s(s_) {}
  ~Scratch() { if (p) cudaFreeAsync(p, s); }
};

static cudaError_t read_flag(const int* err, cudaStream_t s, int* flag) {
  *flag = 0;
  cudaStreamCaptureStatus cs;
  cudaError_t e = cudaStreamIsCapturing(s, &cs);
  if (e != cudaSuccess || cs != cudaStreamCaptureStatusNone) return e;
  e = cudaMemcpyAsync(flag, err, sizeof(int), cudaMemcpyDeviceToHost, s);
  if (e != cudaSuccess) return e;
  return cudaStreamSynchronize(s);
}

static int face_features(const float* pooled, const float* inst, const float* table, const int* rows, int n_labels, int max_rows,
                         int num_images, int feat_num, int table_stride, float* out, int* chosen, int N, int H, int W, int per_image,
                         v2v_stream_t stream) {
  FACE_REQUIRE(pooled && inst && table && rows && out && chosen && N > 0 && H > 0 && W > 0, "face_features: null tensor or empty shape");
  FACE_REQUIRE(n_labels >= 1 && n_labels <= V2V_FACE_MAX_LABELS && feat_num >= 1 && feat_num <= V2V_FACE_MAX_FEAT &&
               table_stride >= feat_num && num_images >= 1 && max_rows >= num_images,
               "face_features: bad table geometry (n_labels %d, feat_num %d, stride %d, num_images %d, max_rows %d)", n_labels,
               feat_num, table_stride, num_images, max_rows);
  FaceFeatParams p{};
  for (int l = 0; l < n_labels; ++l) {
    FACE_REQUIRE(rows[l] >= 0 && rows[l] <= max_rows, "face_features: label %d has %d rows of %d", l, rows[l], max_rows);
    p.rows[l] = rows[l];
  }
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  p.pooled = pooled; p.inst = inst; p.table = table; p.out = out; p.chosen = chosen;
  p.n_labels = n_labels; p.max_rows = max_rows; p.num_images = num_images; p.feat_num = feat_num; p.stride = table_stride;
  p.N = N; p.H = H; p.W = W; p.per_image = per_image;
  const int groups = per_image ? N : 1;
  Scratch sc(s);
  FACE_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&sc.p), sizeof(int) * ((size_t)groups * (FACE_MAX_LABELS + 1) + 1), s));
  FACE_CUDA(cudaMemsetAsync(sc.p, 0x7f, sizeof(int) * (size_t)groups * FACE_MAX_LABELS, s));   // 0x7f7f7f7f: above any flat index
  FACE_CUDA(cudaMemsetAsync(sc.p + (size_t)groups * FACE_MAX_LABELS, 0, sizeof(int) * (groups + 1), s));
  p.first = sc.p; p.bad = sc.p + (size_t)groups * FACE_MAX_LABELS; p.err = p.bad + groups;
  face_first_index_kernel<<<grid_of((size_t)N * H * W), 256, 0, s>>>(p);
  face_choose_kernel<<<groups, 256, 0, s>>>(p);
  face_paint_kernel<<<grid_of((size_t)N * feat_num * H * W), 256, 0, s>>>(p);
  FACE_CUDA(cudaGetLastError());
  int flag;
  FACE_CUDA(read_flag(p.err, s, &flag));
  FACE_REQUIRE(!(flag & FACE_ERR_ID), "face_features: the part map holds a value that is not an integer in [0, %d)", n_labels);
  FACE_REQUIRE(!(flag & FACE_ERR_ROWS), "face_features: a label present in the part map has fewer than num_images = %d rows",
               num_images);
  return 0;
}

}  // namespace v2v

using namespace v2v;

extern "C" {

int v2v_instance_mean(const float* x, const float* inst, float* out, int N, int C, int H, int W, int n_ids, v2v_stream_t stream) {
  FACE_REQUIRE(x && inst && out && N > 0 && C > 0 && H > 0 && W > 0, "instance_mean: null tensor or empty shape");
  FACE_REQUIRE(n_ids >= 1 && n_ids <= V2V_MAX_INSTANCE_IDS, "instance_mean: n_ids %d outside [1, %d]", n_ids, V2V_MAX_INSTANCE_IDS);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  Scratch sc(s);
  FACE_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&sc.p), sizeof(int), s));
  FACE_CUDA(cudaMemsetAsync(sc.p, 0, sizeof(int), s));
  instance_mean_kernel<<<N * C, IM_THREADS, 0, s>>>(x, inst, out, C, H * W, n_ids, sc.p);
  FACE_CUDA(cudaGetLastError());
  int flag;
  FACE_CUDA(read_flag(sc.p, s, &flag));
  FACE_REQUIRE(!(flag & FACE_ERR_ID), "instance_mean: the id map holds a value that is not an integer in [0, %d)", n_ids);
  return 0;
}

int v2v_face_features(const float* pooled, const float* inst, const float* table, const int* rows, int n_labels, int max_rows,
                      int num_images, int feat_num, int table_stride, float* out, int* chosen, int N, int H, int W,
                      v2v_stream_t stream) {
  return face_features(pooled, inst, table, rows, n_labels, max_rows, num_images, feat_num, table_stride, out, chosen, N, H, W, 0,
                       stream);
}

int v2v_face_features_per_image(const float* pooled, const float* inst, const float* table, const int* rows, int n_labels,
                                int max_rows, int num_images, int feat_num, int table_stride, float* out, int* chosen, int N, int H,
                                int W, v2v_stream_t stream) {
  return face_features(pooled, inst, table, rows, n_labels, max_rows, num_images, feat_num, table_stride, out, chosen, N, H, W, 1,
                       stream);
}

}  // extern "C"
