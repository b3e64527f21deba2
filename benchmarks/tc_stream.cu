// Streaming ceilings of the fused predict+score kernel's data path (ffae_tc_kernel), without its MMA chain.
//
// Built and run by benchmarks/bench_tc_stream.py; not part of libgordo_b200.so.  Per window (one row of 64 tags) every
// variant reads x and y and writes the model output (= x here), |x - y|, the same scaled, the same over the feature
// thresholds, and the three row totals: 1 548 bytes.
//   half_row   the kernel's path: persistent grid, three warpgroups, 64-row x / y tiles by TMA (x one tile ahead, y requested
//              after x was read), each per-tag array staged in the warp's two 2 KB slices of the y tile as 16-row x 32-column
//              boxes (both halves of a row staged, then stored together), row totals as plain stores
//   whole_row  the same, but each box is 8 whole rows (one contiguous 2 KB run of HBM): a 3-D tensor map (32 columns, rows,
//              2 halves) keeps the SWIZZLE_128B layout of each half in shared memory
//   plain      full occupancy, float4 loads and stores, no shared memory: the structure-free reference
//
//   tc_stream <windows> <rows per job> <passes> <warmup>     prints one JSON line
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <algorithm>
#include "../gordo_components_b200/csrc/gb_sm90.cuh"

using namespace gb::sm90;

namespace {

constexpr int T = 64, TILE = 64, NWG = 3, NTHREADS = 128 * NWG, BOX_COLS = 32;
constexpr int BOX_BYTES = TILE * BOX_COLS * 4, TILE_BYTES = 2 * BOX_BYTES, OBOX_BYTES = 16 * BOX_COLS * 4;

struct Args {
  CUtensorMap tm_x, tm_y, tm_o[4];
  const float *scale, *ithr;
  float* o[4];
  float *tots, *totu, *totc;
  int rows_per_job, tiles_per_job, n_tiles;
};

__device__ __forceinline__ int box_ofs(int r, int col) { return r * 128 + (((col >> 2) ^ (r & 7)) << 4) + ((col & 3) << 2); }
__device__ __forceinline__ int tile_ofs(int r, int col) { return (col >> 5) * BOX_BYTES + box_ofs(r, col & 31); }

__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, uint32_t src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(map), "r"(src), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}

template <bool WHOLE_ROW>
__global__ void __launch_bounds__(NTHREADS, 1) stream_tc(const __grid_constant__ Args a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ __align__(8) unsigned long long s_bar[2 * NWG];
  __shared__ float vec[2 * T];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wg = warp >> 2, wq = warp & 3, g = lane >> 2, t = lane & 3;
  const uint32_t sbase = smem_u32(smem);
  const uint32_t stage = (sbase + 1023) & ~1023u;
  const uint32_t xbuf = stage + wg * 2 * TILE_BYTES, ybuf = xbuf + TILE_BYTES;
  const uint8_t* xs = smem + (xbuf - sbase);
  const uint8_t* ys = smem + (ybuf - sbase);
  const uint32_t bar_x = smem_u32(&s_bar[wg]), bar_y = smem_u32(&s_bar[NWG + wg]);
  const bool leader = (tid & 127) == 0;
  // the warp's two 2 KB slices of the y tile (its own rows of y).  half_row: box h = rows 16 wq .. of column half h;
  // whole_row: box hr = rows 16 wq + 8 hr .. of both halves, each half a 1 KB SWIZZLE_128B block of 8 rows
  const uint32_t obox0 = ybuf + wq * OBOX_BYTES, obox1 = obox0 + BOX_BYTES;
  if (tid < 2 * T) vec[tid] = tid < T ? a.scale[tid] : a.ithr[tid - T];
  if (tid == 0) {
    for (int i = 0; i < 2 * NWG; ++i) mbar_init(smem_u32(&s_bar[i]), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  uint32_t xp = 0, yp = 0;
  const int stride = gridDim.x * NWG;
  auto row_of = [&](int tile) { return (tile / a.tiles_per_job) * a.rows_per_job + (tile % a.tiles_per_job) * TILE; };
  auto load = [&](const CUtensorMap* m, uint32_t buf, uint32_t bar, int tile) {
    mbar_expect_tx(bar, TILE_BYTES);
    tma_load_2d(buf, m, 0, row_of(tile), bar);
    tma_load_2d(buf + BOX_BYTES, m, BOX_COLS, row_of(tile), bar);
  };
  const int first = blockIdx.x * NWG + wg;
  if (leader && first < a.n_tiles) load(&a.tm_x, xbuf, bar_x, first);
  for (int tile = first; tile < a.n_tiles; tile += stride) {
    float2 xr[2][8], yr[2][8];
    mbar_wait(bar_x, xp);
    xp ^= 1;
#pragma unroll
    for (int hr = 0; hr < 2; ++hr)
#pragma unroll
      for (int j = 0; j < 8; ++j) xr[hr][j] = *reinterpret_cast<const float2*>(xs + tile_ofs(wq * 16 + g + 8 * hr, 8 * j + 2 * t));
    if (lane == 0) bulk_wait_read<0>();
    asm volatile("bar.sync %0, 128;" ::"r"(wg + 1) : "memory");
    if (leader) {
      if (tile + stride < a.n_tiles) load(&a.tm_x, xbuf, bar_x, tile + stride);
      load(&a.tm_y, ybuf, bar_y, tile);
    }
    mbar_wait(bar_y, yp);
    yp ^= 1;
#pragma unroll
    for (int hr = 0; hr < 2; ++hr)
#pragma unroll
      for (int j = 0; j < 8; ++j) yr[hr][j] = *reinterpret_cast<const float2*>(ys + tile_ofs(wq * 16 + g + 8 * hr, 8 * j + 2 * t));
    const int in_job = (tile % a.tiles_per_job) * TILE + wq * 16;  // row inside the job of the warp's first row
    const int orow = row_of(tile) + wq * 16;
    float ss[2] = {0.f, 0.f}, su[2] = {0.f, 0.f};
    if (in_job < a.rows_per_job) {  // (rows per job a multiple of 16: a warp's rows are all live or all past the job)
#pragma unroll
      for (int arr = 0; arr < 4; ++arr) {
        if (arr == 1) {
#pragma unroll
          for (int hr = 0; hr < 2; ++hr)
#pragma unroll
            for (int j = 0; j < 8; ++j) yr[hr][j] = make_float2(fabsf(xr[hr][j].x - yr[hr][j].x), fabsf(xr[hr][j].y - yr[hr][j].y));
        }
        if (arr > 0 && lane == 0) bulk_wait_read<0>();
        __syncwarp();
#pragma unroll
        for (int hr = 0; hr < 2; ++hr)
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int col = 8 * j + 2 * t;
            float2 v = arr == 0 ? xr[hr][j] : yr[hr][j];
            if (arr > 1) {
              const float2 s = *reinterpret_cast<const float2*>(vec + (arr == 3 ? T : 0) + col);
              v = make_float2(v.x * s.x, v.y * s.y);
            }
            if (arr == 1) su[hr] += v.x * v.x + v.y * v.y;
            if (arr == 2) ss[hr] += v.x * v.x + v.y * v.y;
            const uint32_t box = (WHOLE_ROW ? hr : j >> 2) ? obox1 : obox0;
            const int ofs = WHOLE_ROW ? (j >> 2) * 1024 + box_ofs(g, col & 31) : box_ofs(g + 8 * hr, col & 31);
            *reinterpret_cast<float2*>(smem + (box - sbase) + ofs) = v;
          }
        fence_proxy_async();
        __syncwarp();
        if (lane == 0) {
          if (WHOLE_ROW) {
            tma_store_3d(&a.tm_o[arr], obox0, 0, orow, 0);
            tma_store_3d(&a.tm_o[arr], obox1, 0, orow + 8, 0);
          } else {
            tma_store_2d(&a.tm_o[arr], obox0, 0, orow);
            tma_store_2d(&a.tm_o[arr], obox1, BOX_COLS, orow);
          }
          bulk_commit();
        }
      }
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        ss[hr] += __shfl_xor_sync(0xffffffffu, ss[hr], 1);
        ss[hr] += __shfl_xor_sync(0xffffffffu, ss[hr], 2);
        su[hr] += __shfl_xor_sync(0xffffffffu, su[hr], 1);
        su[hr] += __shfl_xor_sync(0xffffffffu, su[hr], 2);
        if (t == 0) {
          const long r = orow + g + 8 * hr;
          a.tots[r] = ss[hr] * (1.f / T);
          a.totu[r] = su[hr] * (1.f / T);
          a.totc[r] = ss[hr] * (1.f / T) * 20.f;
        }
      }
    }
  }
  if (lane == 0) bulk_wait<0>();
}

// 16 threads per row, one float4 of x and y each; row totals by shuffles within the 16
__global__ void __launch_bounds__(256) stream_plain(const float4* __restrict__ x, const float4* __restrict__ y, const float* __restrict__ scale,
                                                    const float* __restrict__ ithr, float4* o0, float4* o1, float4* o2, float4* o3, float* tots,
                                                    float* totu, float* totc, long n_rows) {
  const int c = threadIdx.x & 15;
  const float4 s = reinterpret_cast<const float4*>(scale)[c], it = reinterpret_cast<const float4*>(ithr)[c];
  for (long r = (blockIdx.x * (long)blockDim.x + threadIdx.x) >> 4; r < n_rows; r += ((long)gridDim.x * blockDim.x) >> 4) {
    const long i = r * 16 + c;
    const float4 xv = __ldcs(x + i), yv = __ldcs(y + i);
    const float4 df = make_float4(fabsf(xv.x - yv.x), fabsf(xv.y - yv.y), fabsf(xv.z - yv.z), fabsf(xv.w - yv.w));
    const float4 e = make_float4(df.x * s.x, df.y * s.y, df.z * s.z, df.w * s.w);
    __stcs(o0 + i, xv);
    __stcs(o1 + i, df);
    __stcs(o2 + i, e);
    __stcs(o3 + i, make_float4(df.x * it.x, df.y * it.y, df.z * it.z, df.w * it.w));
    float su = df.x * df.x + df.y * df.y + df.z * df.z + df.w * df.w, ss = e.x * e.x + e.y * e.y + e.z * e.z + e.w * e.w;
#pragma unroll
    for (int m = 1; m < 16; m <<= 1) {
      su += __shfl_xor_sync(0xffffffffu, su, m);
      ss += __shfl_xor_sync(0xffffffffu, ss, m);
    }
    if (c == 0) {
      tots[r] = ss * (1.f / T);
      totu[r] = su * (1.f / T);
      totc[r] = ss * (1.f / T) * 20.f;
    }
  }
}

__global__ void fill(float* p, long n, unsigned seed) {
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    unsigned h = (unsigned)i * 2654435761u ^ seed;
    h ^= h >> 15; h *= 2246822519u; h ^= h >> 13;
    p[i] = (float)(h & 0xffffff) * (1.f / 16777216.f);
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// [rows][64] fp32 as (32 columns, rows, 2 halves): strides 256 B for rows, 128 B for halves; boxes of 32 x 8 x 2
CUresult encode_whole_row(CUtensorMap* map, float* base, long rows) {
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
    return CUDA_ERROR_NOT_FOUND;
  const cuuint64_t dims[3] = {BOX_COLS, (cuuint64_t)rows, 2};
  const cuuint64_t strides[2] = {T * 4, BOX_COLS * 4};
  const cuuint32_t box[3] = {BOX_COLS, 8, 2};
  const cuuint32_t estr[3] = {1, 1, 1};
  return reinterpret_cast<EncodeTiledFn>(p)(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

#define CK(x)                                                                                   \
  do {                                                                                          \
    cudaError_t e_ = (x);                                                                       \
    if (e_ != cudaSuccess) {                                                                    \
      fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_));        \
      exit(1);                                                                                  \
    }                                                                                           \
  } while (0)

}  // namespace

int main(int argc, char** argv) {
  const long windows = argc > 1 ? atol(argv[1]) : 10000000L;
  const int rows_per_job = argc > 2 ? atoi(argv[2]) : 10000;
  const int passes = argc > 3 ? atoi(argv[3]) : 20, warmup = argc > 4 ? atoi(argv[4]) : 3;
  if (rows_per_job % 16 || windows % rows_per_job) {
    fprintf(stderr, "rows per job must be a multiple of 16 and divide the windows\n");
    return 2;
  }
  int sms = 0;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  const long n = windows * T;
  float *x, *y, *vecs, *o[4], *tot;
  CK(cudaMalloc(&x, n * 4));
  CK(cudaMalloc(&y, n * 4));
  for (auto& p : o) CK(cudaMalloc(&p, n * 4));
  CK(cudaMalloc(&tot, 3 * windows * 4));
  CK(cudaMalloc(&vecs, 2 * T * 4));
  fill<<<1024, 256>>>(x, n, 1u);
  fill<<<1024, 256>>>(y, n, 2u);
  fill<<<1, 128>>>(vecs, 2 * T, 3u);
  CK(cudaGetLastError());

  Args a{};
  a.scale = vecs; a.ithr = vecs + T;
  for (int i = 0; i < 4; ++i) a.o[i] = o[i];
  a.tots = tot; a.totu = tot + windows; a.totc = tot + 2 * windows;
  a.rows_per_job = rows_per_job;
  a.tiles_per_job = (rows_per_job + TILE - 1) / TILE;
  a.n_tiles = (int)(windows / rows_per_job) * a.tiles_per_job;
  const size_t smem = 1024 + NWG * 2 * TILE_BYTES;

  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  auto time = [&](auto launch) {
    for (int i = 0; i < warmup; ++i) launch();
    CK(cudaDeviceSynchronize());
    std::vector<float> ms(passes);
    for (int i = 0; i < passes; ++i) {
      CK(cudaEventRecord(e0));
      launch();
      CK(cudaEventRecord(e1));
      CK(cudaEventSynchronize(e1));
      CK(cudaEventElapsedTime(&ms[i], e0, e1));
    }
    CK(cudaGetLastError());
    std::sort(ms.begin(), ms.end());
    double mean = 0;
    for (float v : ms) mean += v;
    return std::vector<double>{mean / passes, ms.front(), ms.back()};
  };
  const double bytes = 1548.0 * windows;
  printf("{\"windows\": %ld, \"rows_per_job\": %d, \"passes\": %d, \"bytes_per_window\": 1548", windows, rows_per_job, passes);
  auto report = [&](const char* name, std::vector<double> r) {
    printf(", \"%s\": {\"ms\": %.4f, \"ms_min\": %.4f, \"ms_max\": %.4f, \"GBps\": %.1f}", name, r[0], r[1], r[2], bytes / (r[0] * 1e6));
  };

  CUresult cr = gb::sm90::encode_map_2d(&a.tm_x, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, x, windows, T, BOX_COLS, TILE);
  if (cr == CUDA_SUCCESS) cr = gb::sm90::encode_map_2d(&a.tm_y, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, y, windows, T, BOX_COLS, TILE);
  for (int i = 0; i < 4 && cr == CUDA_SUCCESS; ++i) cr = gb::sm90::encode_map_2d(&a.tm_o[i], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, o[i], windows, T, BOX_COLS, 16);
  if (cr != CUDA_SUCCESS) {
    fprintf(stderr, "cuTensorMapEncodeTiled failed: %d\n", (int)cr);
    return 1;
  }
  CK(cudaFuncSetAttribute(stream_tc<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  CK(cudaFuncSetAttribute(stream_tc<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  report("half_row", time([&] { stream_tc<false><<<sms, NTHREADS, smem>>>(a); }));

  for (int i = 0; i < 4 && cr == CUDA_SUCCESS; ++i) cr = encode_whole_row(&a.tm_o[i], o[i], windows);
  if (cr == CUDA_SUCCESS)
    report("whole_row", time([&] { stream_tc<true><<<sms, NTHREADS, smem>>>(a); }));
  else
    printf(", \"whole_row\": {\"error\": \"cuTensorMapEncodeTiled refused the (columns, rows, halves) map: CUresult %d\"}", (int)cr);

  int plain_blocks = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&plain_blocks, stream_plain, 256, 0));
  report("plain", time([&] {
           stream_plain<<<sms * plain_blocks, 256>>>((const float4*)x, (const float4*)y, vecs, vecs + T, (float4*)o[0], (float4*)o[1], (float4*)o[2],
                                                      (float4*)o[3], a.tots, a.totu, a.totc, windows);
         }));
  printf("}\n");
  return 0;
}
