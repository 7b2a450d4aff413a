// The fixed-order CTA reduction of the loss, metric and evaluation kernels (DESIGN §4.12).  No atomics: the tree
// and the thread count fix the association of every sum, so a result is identical bit for bit from run to run.
#pragma once

namespace srcv {

// Fixed-order CTA reduction: after a barrier, for o = kThreads/2 .. 1 thread t < o calls fold(t, t + o),
// with a barrier after each step.  On return slot 0 holds the total, visible to every thread.
template <int kThreads, class Fold>
__device__ __forceinline__ void block_tree(Fold fold) {
  __syncthreads();
  for (int o = kThreads / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) fold((int)threadIdx.x, (int)threadIdx.x + o);
    __syncthreads();
  }
}

// One CTA sums the partials [p0, p1) of psum, and of pcnt unless it is null, in a fixed order: thread-strided,
// then block_tree.  On return s_sum[0] and s_cnt[0] hold the totals.  The barrier before the shared writes lets a
// caller loop without a barrier of its own after reading the previous totals.
template <int kThreads>
__device__ __forceinline__ void reduce_partials(const double* psum, const long long* pcnt, unsigned p0, unsigned p1,
                                                double* s_sum, long long* s_cnt) {
  double sum = 0.0;
  long long cnt = 0;
  for (unsigned i = p0 + threadIdx.x; i < p1; i += kThreads) {
    sum += psum[i];
    if (pcnt) cnt += pcnt[i];
  }
  __syncthreads();
  s_sum[threadIdx.x] = sum;
  s_cnt[threadIdx.x] = cnt;
  block_tree<kThreads>([&](int t, int u) {
    s_sum[t] += s_sum[u];
    s_cnt[t] += s_cnt[u];
  });
}

}  // namespace srcv
