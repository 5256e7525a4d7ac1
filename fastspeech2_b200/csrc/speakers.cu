// Speaker table of the train step (DESIGN.md section 25): the broadcast add y = x + table[spk[b]] over every row of an
// utterance, and its backward into the table.  The eval path fuses the same add into the last encoder LayerNorm
// (rowwise.cu, RowNorm::spk_table); here it stands alone because the train step's LayerNorm is its own autograd stage.
//
// The backward has no floating-point atomics.  Up to B*T rows land on at most B table rows, so an atomicAdd per row (as
// embed_backward does for phonemes) would contend on a handful of addresses and round in a different order every run.
// Instead:
//   stage 1: one CTA per (utterance, 32 columns): 8 row lanes sum rows t = lane, lane + 8, ... in order, then a fixed
//            three-level tree over the lanes -> part[b][c];
//   stage 2: one thread per (utterance b, column c) where b is the first utterance of its speaker: it sums the partials
//            of every utterance of that speaker in ascending b and adds the total to dtable[spk][c] once.
// Both orders depend only on the shapes, so the same dy always gives the same bits.
#include "common.cuh"

namespace fs2 {
namespace {

constexpr int SPK_COLS = 32, SPK_LANES = 8;

__global__ void speaker_add_kernel(const float4* __restrict__ x, const int64_t* __restrict__ spk, const float4* __restrict__ table,
                                   int T, int C4, int n, float4* __restrict__ y, long total) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long row = i / C4;
    const int c = (int)(i - row * C4);
    const int64_t id = __ldg(spk + row / T);
    float4 v = x[i];
    if (id >= 0 && id < n) {
      const float4 e = __ldg(table + id * C4 + c);
      v.x = __fadd_rn(v.x, e.x); v.y = __fadd_rn(v.y, e.y); v.z = __fadd_rn(v.z, e.z); v.w = __fadd_rn(v.w, e.w);
    }
    y[i] = v;
  }
}

// grid (ceil(C / 32), B), block (32, 8)
__global__ void speaker_colsum_kernel(const float* __restrict__ dy, int T, int C, float* __restrict__ part) {
  __shared__ float s[SPK_LANES][SPK_COLS];
  const int b = blockIdx.y, c = blockIdx.x * SPK_COLS + threadIdx.x, lane = threadIdx.y;
  float acc = 0.f;
  if (c < C)
    for (int t = lane; t < T; t += SPK_LANES) acc += dy[((long)b * T + t) * C + c];
  s[lane][threadIdx.x] = acc;
  __syncthreads();
#pragma unroll
  for (int h = SPK_LANES / 2; h > 0; h >>= 1) {
    if (lane < h) s[lane][threadIdx.x] += s[lane + h][threadIdx.x];
    __syncthreads();
  }
  if (lane == 0 && c < C) part[(long)b * C + c] = s[0][threadIdx.x];
}

__global__ void speaker_scatter_kernel(const float* __restrict__ part, const int64_t* __restrict__ spk, int B, int C, int n,
                                       float* __restrict__ dtable) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)B * C) return;
  const int b = (int)(i / C), c = (int)(i - (long)b * C);
  const int64_t id = spk[b];
  if (id < 0 || id >= n) return;
  for (int k = 0; k < b; ++k)
    if (spk[k] == id) return;                 // not the first utterance of this speaker: that one's thread owns the row
  float acc = part[(long)b * C + c];
  for (int k = b + 1; k < B; ++k)
    if (spk[k] == id) acc += part[(long)k * C + c];
  dtable[id * C + c] += acc;
}

}  // namespace
}  // namespace fs2

using namespace fs2;

extern "C" {

int fs2_speaker_add(const float* x, const int64_t* spk, const float* table, int B, int T, int C, int n, float* y, void* stream) {
  FS2_REQUIRE(x && spk && table && y, "fs2_speaker_add: null argument");
  FS2_REQUIRE(B >= 0 && T >= 0 && C > 0 && C % 4 == 0 && n >= 1, "fs2_speaker_add: bad shape B=%d T=%d C=%d n=%d", B, T, C, n);
  FS2_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(table)) & 15) == 0,
              "fs2_speaker_add: x, table and y must be 16-byte aligned");
  const long total = (long)B * T * (C / 4);
  if (total == 0) return FS2_OK;
  speaker_add_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const float4*>(x), spk, reinterpret_cast<const float4*>(table), T, C / 4, n, reinterpret_cast<float4*>(y), total);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

int fs2_speaker_add_backward_ws_bytes(int B, int C, size_t* bytes) {
  FS2_REQUIRE(bytes && B >= 0 && C > 0, "fs2_speaker_add_backward_ws_bytes: bad argument");
  *bytes = align256((size_t)B * C * sizeof(float));
  return FS2_OK;
}

int fs2_speaker_add_backward(const float* dy, const int64_t* spk, int B, int T, int C, int n, float* dtable, void* ws,
                             size_t ws_bytes, void* stream) {
  FS2_REQUIRE(dy && spk && dtable && (ws || B == 0), "fs2_speaker_add_backward: null argument");
  FS2_REQUIRE(B >= 0 && T >= 0 && C > 0 && n >= 1 && B <= 65535, "fs2_speaker_add_backward: bad shape B=%d T=%d C=%d n=%d", B, T, C, n);
  FS2_REQUIRE(ws_bytes >= (size_t)B * C * sizeof(float), "fs2_speaker_add_backward: workspace too small (%zu < %zu)", ws_bytes,
              (size_t)B * C * sizeof(float));
  if (B == 0) return FS2_OK;
  cudaStream_t st = (cudaStream_t)stream;
  float* part = reinterpret_cast<float*>(ws);
  speaker_colsum_kernel<<<dim3((C + SPK_COLS - 1) / SPK_COLS, B), dim3(SPK_COLS, SPK_LANES), 0, st>>>(dy, T, C, part);
  FS2_LAUNCH_CHECK();
  const long cells = (long)B * C;
  speaker_scatter_kernel<<<(int)((cells + 255) / 256), 256, 0, st>>>(part, spk, B, C, n, dtable);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

}  // extern "C"
