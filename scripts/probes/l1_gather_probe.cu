// L1 data-pipe ceiling for the access shape of the dot sweep — a measurement tool, not product.
//
// The dot-product sweep (csrc/srcv_dot.cu) is bound by the L1/shared-memory data pipe, not by
// HBM (DESIGN.md §4.2): every (plane, view, pixel) sample pulls 4 taps x 64 B through L1 with
// warp-wide LDG.128 whose 16 lanes per row read a 256-byte row segment at an arbitrary 16-byte
// offset.  This probe issues exactly that load shape from an L1-resident window with no
// arithmetic beyond keeping the values alive, and reports bytes per clock per SM, so that the
// sweep's achieved L1 rate has a MEASURED denominator next to the nominal 128 B/clk/SM.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o scripts/probes/l1_gather_probe scripts/probes/l1_gather_probe.cu
//   ./scripts/probes/l1_gather_probe            (prints one JSON line per access shape)
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

constexpr int kW = 160, kH = 24;          // texel window per CTA: 160 x 24 x 16 B = 60 KB (L1-resident)
constexpr int kIters = 4096;

// tile_w = 16: lane -> (lane & 15, lane >> 4) like the sweep's 16x2 warp tile; 32: one 32-pixel row.
// step16 = texel offset added per iteration (1 = walks through every 16-byte alignment).
template <int TILE_W>
__global__ void __launch_bounds__(64) probe(const float4* __restrict__ win, float4* __restrict__ sink,
                                            int step16, long long* __restrict__ cycles) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int lx = lane & (TILE_W - 1), ly = lane / TILE_W;
  const float4* base = win + (size_t)blockIdx.x % 4 * 0;   // every CTA reads the same window (L1/L2 hot)
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  int x = warp * 3, y = warp * 5;
  // warm the window into L1
  for (int i = threadIdx.x; i < kW * kH; i += blockDim.x) { const float4 v = __ldg(base + i); acc.x += v.x; }
  __syncthreads();
  const long long t0 = clock64();
#pragma unroll 1
  for (int it = 0; it < kIters; ++it) {
    // the four taps of one bilinear footprint: (x, y), (x+1, y), (x, y+1), (x+1, y+1)
    const float4* q = base + (y + ly) * kW + x + lx;
    const float4 a = __ldg(q), b = __ldg(q + 1), c = __ldg(q + kW), d = __ldg(q + kW + 1);
    // every component is consumed so the loads stay 16-byte vector loads (16 FADD per 4 LDG.128)
    acc.x += (a.x + b.x) + (c.x + d.x); acc.y += (a.y + b.y) + (c.y + d.y);
    acc.z += (a.z + b.z) + (c.z + d.z); acc.w += (a.w + b.w) + (c.w + d.w);
    x += step16; if (x > kW - TILE_W - 2) x -= kW - TILE_W - 2;
    y += 1; if (y > kH - 4) y = 0;
  }
  const long long t1 = clock64();
  sink[blockIdx.x * blockDim.x + threadIdx.x] = acc;
  if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

template <int TILE_W>
static void run(const char* name, int step16, int ctas_per_sm, int sms, const float4* win, float4* sink,
                long long* cycles_d) {
  const int grid = sms * ctas_per_sm;
  probe<TILE_W><<<grid, 64>>>(win, sink, step16, cycles_d);
  cudaDeviceSynchronize();
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0);
  probe<TILE_W><<<grid, 64>>>(win, sink, step16, cycles_d);
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  float ms = 0.f;
  cudaEventElapsedTime(&ms, e0, e1);
  long long* h = (long long*)malloc(sizeof(long long) * grid);
  cudaMemcpy(h, cycles_d, sizeof(long long) * grid, cudaMemcpyDeviceToHost);
  double mean = 0;
  for (int i = 0; i < grid; ++i) mean += (double)h[i];
  mean /= grid;
  free(h);
  // bytes requested per CTA: 2 warps x kIters x 4 taps x 512 B; CTAs of one SM run concurrently
  const double bytes_per_sm = (double)ctas_per_sm * 2 * kIters * 4 * 512;
  printf("{\"probe\": \"l1_gather\", \"shape\": \"%s\", \"step_texels\": %d, \"warps_per_sm\": %d, "
         "\"bytes_per_clk_per_sm\": %.1f, \"kernel_ms\": %.3f, \"err\": \"%s\"}\n",
         name, step16, ctas_per_sm * 2, bytes_per_sm / mean, ms, cudaGetErrorString(cudaGetLastError()));
}

int main() {
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  float4 *win, *sink;
  long long* cyc;
  cudaMalloc(&win, sizeof(float4) * kW * kH);
  cudaMemset(win, 0, sizeof(float4) * kW * kH);
  cudaMalloc(&sink, sizeof(float4) * 64 * sms * 32);
  cudaMalloc(&cyc, sizeof(long long) * sms * 32);
  for (int occ : {8, 16, 32}) {           // 16, 32, 64 warps per SM
    run<16>("16x2_tile", 1, occ, sms, win, sink, cyc);   // every 16-byte alignment: the sweep's shape
    run<16>("16x2_tile_aligned", 8, occ, sms, win, sink, cyc);   // row segments stay 128-byte aligned
    run<32>("32x1_tile", 1, occ, sms, win, sink, cyc);
  }
  return 0;
}
