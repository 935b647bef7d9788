// Device helpers shared by the tree fits (forest.cu, gbrt.cu).
#pragma once

// Stable partition of one segment seg[0, c) by pred, by one warp: lefts in place (a left is never written past the positions the
// warp has read), rights through tr[] and back.  Returns the left count.
template <typename P>
__device__ __forceinline__ int warp_partition(int* seg, int* tr, int c, P pred) {
  const int lane = threadIdx.x & 31;
  const unsigned lt = (1u << lane) - 1u;
  int nl = 0, nr = 0;
  for (int j0 = 0; j0 < c; j0 += 32) {
    const int j = j0 + lane;
    const bool valid = j < c;
    const int i = valid ? seg[j] : 0;
    const bool L = valid && pred(i), R = valid && !L;
    __syncwarp();
    const unsigned ml = __ballot_sync(0xffffffffu, L), mr = __ballot_sync(0xffffffffu, R);
    if (L) seg[nl + __popc(ml & lt)] = i;
    if (R) tr[nr + __popc(mr & lt)] = i;
    nl += __popc(ml);
    nr += __popc(mr);
  }
  __syncwarp();
  for (int j = lane; j < nr; j += 32) seg[nl + j] = tr[j];
  __syncwarp();
  return nl;
}
