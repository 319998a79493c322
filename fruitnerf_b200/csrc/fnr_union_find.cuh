// Lock-free union-find over int indices, shared by DBSCAN (fnr_cluster.cu) and the chart unwrap (fnr_unwrap.cu).
// parent[i] <= i always holds (a root is only ever hooked under a smaller root), so the root of a component is its
// smallest index whatever order the CAS operations land in.
#pragma once

namespace fnr {

__device__ __forceinline__ int find_root(volatile int* parent, int i) {
  int cur = parent[i];
  if (cur != i) {
    int prev = i, next;
    while (cur > (next = parent[cur])) {  // path halving; a stale read only sees a larger (still valid) ancestor
      parent[prev] = next;
      prev = cur;
      cur = next;
    }
  }
  return cur;
}

__device__ __forceinline__ void unite(int* parent, int a, int b) {
  int ra = find_root(parent, a), rb = find_root(parent, b);
  while (ra != rb) {
    const int lo = min(ra, rb), hi = max(ra, rb);
    const int old = atomicCAS(parent + hi, hi, lo);
    if (old == hi) return;
    ra = find_root(parent, old);
    rb = find_root(parent, lo);
  }
}

}  // namespace fnr
