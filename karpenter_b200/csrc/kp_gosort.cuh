// kp_gosort.cuh -- Go's sort.Slice (pdqsort_func of package sort, go1.26) on the claim-order arrays, executed by one
// warp.
//
// Emulated exactly because the permutation it leaves among claims with EQUAL pod counts decides first-fit
// (scheduler.go:504).  key = len(Pods) by position, val = claim id by position.  The control flow is Go's, statement
// for statement, and is warp-uniform; what the warp parallelises are the linear scans inside it (the two-pointer
// partition loops, the "first inversion" search of partialInsertionSort, the element shifts, insertion sort of <= 12
// elements as a stable rank computation), each a 32-wide compare + ballot instead of a scalar loop.
#pragma once
#include <cuda_runtime.h>

#ifndef FULL
#define FULL 0xffffffffu
#endif

// PM: a second payload by position, moved with `val` (the claim order's failure masks)
template <class K, bool PM = false>
struct WarpSorterT {
  K* key;    // sort key by position (pod count of a claim; price of an instance type)
  int* val;  // payload by position
  int lane;
  ulonglong2* pm;

  __device__ bool less(int i, int j) const { return key[i] < key[j]; }
  __device__ void swap(int i, int j) {
    if (lane == 0) {
      K tk = key[i];
      key[i] = key[j];
      key[j] = tk;
      int t = val[i];
      val[i] = val[j];
      val[j] = t;
      if (PM) {
        const ulonglong2 tp = pm[i];
        pm[i] = pm[j];
        pm[j] = tp;
      }
    }
    __syncwarp();
  }
  // smallest idx in [i, j] whose key is NOT < pv (j + 1 if none):   for i <= j && less(i, a) { i++ }
  __device__ int first_not_less(int i, int j, K pv) const {
    for (int b = i; b <= j; b += 32) {
      int idx = b + lane;
      unsigned m = __ballot_sync(FULL, idx <= j && !(key[idx] < pv));
      if (m) return b + __ffs(m) - 1;
    }
    return j + 1;
  }
  // largest idx in [i, j] whose key IS < pv (i - 1 if none):        for i <= j && !less(j, a) { j-- }
  __device__ int last_less(int i, int j, K pv) const {
    for (int b = j; b >= i; b -= 32) {
      int idx = b - lane;
      unsigned m = __ballot_sync(FULL, idx >= i && key[idx] < pv);
      if (m) return b - (__ffs(m) - 1);
    }
    return i - 1;
  }
  // smallest idx in [i, j] with pv < key[idx] (j + 1 if none):      for i <= j && !less(a, i) { i++ }
  __device__ int first_greater(int i, int j, K pv) const {
    for (int b = i; b <= j; b += 32) {
      int idx = b + lane;
      unsigned m = __ballot_sync(FULL, idx <= j && pv < key[idx]);
      if (m) return b + __ffs(m) - 1;
    }
    return j + 1;
  }
  // largest idx in [i, j] with !(pv < key[idx]) (i - 1 if none):    for i <= j && less(a, j) { j-- }
  __device__ int last_not_greater(int i, int j, K pv) const {
    for (int b = j; b >= i; b -= 32) {
      int idx = b - lane;
      unsigned m = __ballot_sync(FULL, idx >= i && !(pv < key[idx]));
      if (m) return b - (__ffs(m) - 1);
    }
    return i - 1;
  }
  // move element `from` to position `to` (to < from), shifting [to, from) right by one
  __device__ void rotate_right(int to, int from) {
    const K ek = key[from];
    const int ev = val[from];
    ulonglong2 ep = {};
    if (PM) ep = pm[from];
    for (int b0 = from; b0 > to; b0 -= 32) {
      const int i = b0 - lane;
      K vk = 0;
      int vv = 0;
      ulonglong2 vp = {};
      if (i > to) {
        vk = key[i - 1];
        vv = val[i - 1];
        if (PM) vp = pm[i - 1];
      }
      __syncwarp();
      if (i > to) {
        key[i] = vk;
        val[i] = vv;
        if (PM) pm[i] = vp;
      }
      __syncwarp();
    }
    if (lane == 0) {
      key[to] = ek;
      val[to] = ev;
      if (PM) pm[to] = ep;
    }
    __syncwarp();
  }
  // move element `from` to position `to` (to > from), shifting (from, to] left by one
  __device__ void rotate_left(int from, int to) {
    const K ek = key[from];
    const int ev = val[from];
    ulonglong2 ep = {};
    if (PM) ep = pm[from];
    for (int b0 = from; b0 < to; b0 += 32) {
      const int i = b0 + lane;
      K vk = 0;
      int vv = 0;
      ulonglong2 vp = {};
      if (i < to) {
        vk = key[i + 1];
        vv = val[i + 1];
        if (PM) vp = pm[i + 1];
      }
      __syncwarp();
      if (i < to) {
        key[i] = vk;
        val[i] = vv;
        if (PM) pm[i] = vp;
      }
      __syncwarp();
    }
    if (lane == 0) {
      key[to] = ek;
      val[to] = ev;
      if (PM) pm[to] = ep;
    }
    __syncwarp();
  }
  // insertionSortCmpFunc on [a, b), b - a <= 32: insertion sort is stable, so the result is the stable rank order
  __device__ void insertion_sort(int a, int b) {
    const int n = b - a;
    K k = 0;
    int v = 0;
    ulonglong2 p = {};
    if (lane < n) {
      k = key[a + lane];
      v = val[a + lane];
      if (PM) p = pm[a + lane];
    }
    int rank = 0;
    for (int j = 0; j < n; j++) {
      const K kj = __shfl_sync(FULL, k, j);
      rank += (kj < k || (kj == k && j < lane)) ? 1 : 0;
    }
    __syncwarp();
    if (lane < n) {
      key[a + rank] = k;
      val[a + rank] = v;
      if (PM) pm[a + rank] = p;
    }
    __syncwarp();
  }
  __device__ void sift_down(int lo, int hi, int first) {
    int root = lo;
    for (;;) {
      int child = 2 * root + 1;
      if (child >= hi) return;
      if (child + 1 < hi && less(first + child, first + child + 1)) child++;
      if (!less(first + root, first + child)) return;
      swap(first + root, first + child);
      root = child;
    }
  }
  __device__ void heap_sort(int a, int b) {
    int first = a, lo = 0, hi = b - a;
    for (int i = (hi - 1) / 2; i >= 0; i--) sift_down(i, hi, first);
    for (int i = hi - 1; i >= 0; i--) {
      swap(first, first + i);
      sift_down(lo, i, first);
    }
  }
  __device__ int partition(int a, int b, int pivot, bool* already) {
    swap(a, pivot);
    const K pv = key[a];
    int i = a + 1, j = b - 1;
    i = first_not_less(i, j, pv);
    j = last_less(i, j, pv);
    if (i > j) {
      swap(j, a);
      *already = true;
      return j;
    }
    swap(i, j);
    i++;
    j--;
    for (;;) {
      i = first_not_less(i, j, pv);
      j = last_less(i, j, pv);
      if (i > j) break;
      swap(i, j);
      i++;
      j--;
    }
    swap(j, a);
    *already = false;
    return j;
  }
  __device__ int partition_equal(int a, int b, int pivot) {
    swap(a, pivot);
    const K pv = key[a];
    int i = a + 1, j = b - 1;
    for (;;) {
      i = first_greater(i, j, pv);
      j = last_not_greater(i, j, pv);
      if (i > j) break;
      swap(i, j);
      i++;
      j--;
    }
    return i;
  }
  __device__ bool partial_insertion_sort(int a, int b) {
    int i = a + 1;
    for (int j = 0; j < 5; j++) {
      {  // for i < b && !less(i, i-1) { i++ }
        int found = b;
        for (int b0 = i; b0 < b; b0 += 32) {
          int idx = b0 + lane;
          unsigned m = __ballot_sync(FULL, idx < b && key[idx] < key[idx - 1]);
          if (m) {
            found = b0 + __ffs(m) - 1;
            break;
          }
        }
        i = found;
      }
      if (i == b) return true;
      if (b - a < 50) return false;
      swap(i, i - 1);
      if (i - a >= 2) {  // shift the smaller one to the left:  for j := i-1; j >= 1; j-- { if !less(j, j-1) break; swap }
        const K x = key[i - 1];
        int stop = last_not_greater_from(i - 2, x);  // largest m in [0, i-2] with key[m] <= x, else -1
        if (stop + 1 < i - 1) rotate_right(stop + 1, i - 1);
      }
      if (b - i >= 2) {  // shift the greater one to the right: for j := i+1; j < b; j++ { if !less(j, j-1) break; swap }
        const K x = key[i];
        int stop = b;  // smallest m in [i+1, b) with !(key[m] < x), else b
        for (int b0 = i + 1; b0 < b; b0 += 32) {
          int idx = b0 + lane;
          unsigned m = __ballot_sync(FULL, idx < b && !(key[idx] < x));
          if (m) {
            stop = b0 + __ffs(m) - 1;
            break;
          }
        }
        if (stop - 1 > i) rotate_left(i, stop - 1);
      }
    }
    return false;
  }
  // largest m in [0, hi] with key[m] <= x, else -1
  __device__ int last_not_greater_from(int hi, K x) const {
    for (int b = hi; b >= 0; b -= 32) {
      int idx = b - lane;
      unsigned m = __ballot_sync(FULL, idx >= 0 && !(x < key[idx]));
      if (m) return b - (__ffs(m) - 1);
    }
    return -1;
  }
  __device__ static int bits_len(unsigned long long x) { return x ? 64 - __clzll((long long)x) : 0; }
  __device__ void break_patterns(int a, int b) {
    int length = b - a;
    if (length >= 8) {
      unsigned long long random = (unsigned long long)length;
      unsigned long long modulus = 1ull << bits_len((unsigned long long)length);
      int idx = a + (length / 4) * 2 - 1;
      for (int i = 0; i < 3; i++) {
        random ^= random << 13;
        random ^= random >> 7;
        random ^= random << 17;
        int other = (int)(random & (modulus - 1));
        if (other >= length) other -= length;
        swap(idx - 1 + i, a + other);
      }
    }
  }
  __device__ void order2(int* a, int* b, int* swaps) const {
    if (less(*b, *a)) {
      (*swaps)++;
      int t = *a;
      *a = *b;
      *b = t;
    }
  }
  __device__ int median(int a, int b, int c, int* swaps) const {
    order2(&a, &b, swaps);
    order2(&b, &c, swaps);
    order2(&a, &b, swaps);
    return b;
  }
  // returns pivot; hint: 0 unknown, 1 increasing, 2 decreasing
  __device__ int choose_pivot(int a, int b, int* hint) const {
    int l = b - a, swaps = 0;
    int i = a + l / 4 * 1, j = a + l / 4 * 2, k = a + l / 4 * 3;
    if (l >= 8) {
      if (l >= 50) {
        i = median(i - 1, i, i + 1, &swaps);
        j = median(j - 1, j, j + 1, &swaps);
        k = median(k - 1, k, k + 1, &swaps);
      }
      j = median(i, j, k, &swaps);
    }
    *hint = swaps == 0 ? 1 : (swaps == 12 ? 2 : 0);
    return j;
  }
  __device__ void reverse_range(int a, int b) {
    const int n = b - a;
    for (int b0 = 0; b0 < n / 2; b0 += 32) {
      const int t = b0 + lane;
      if (t < n / 2) {
        const int i = a + t, j = b - 1 - t;
        K tk = key[i];
        int tv = val[i];
        key[i] = key[j];
        val[i] = val[j];
        key[j] = tk;
        val[j] = tv;
        if (PM) {
          const ulonglong2 tp = pm[i];
          pm[i] = pm[j];
          pm[j] = tp;
        }
      }
    }
    __syncwarp();
  }
  __device__ void pdqsort(int a, int b, int limit) {
    bool wasBalanced = true, wasPartitioned = true;
    for (;;) {
      int length = b - a;
      if (length <= 12) {
        insertion_sort(a, b);
        return;
      }
      if (limit == 0) {
        heap_sort(a, b);
        return;
      }
      if (!wasBalanced) {
        break_patterns(a, b);
        limit--;
      }
      int hint;
      int pivot = choose_pivot(a, b, &hint);
      if (hint == 2) {
        reverse_range(a, b);
        pivot = (b - 1) - (pivot - a);
        hint = 1;
      }
      if (wasBalanced && wasPartitioned && hint == 1) {
        if (partial_insertion_sort(a, b)) return;
      }
      if (a > 0 && !less(a - 1, pivot)) {
        a = partition_equal(a, b, pivot);
        continue;
      }
      bool already;
      int mid = partition(a, b, pivot, &already);
      wasPartitioned = already;
      int leftLen = mid - a, rightLen = b - mid;
      int balanceThreshold = length / 8;
      if (leftLen < rightLen) {
        wasBalanced = leftLen >= balanceThreshold;
        pdqsort(a, mid, limit);
        a = mid + 1;
      } else {
        wasBalanced = rightLen >= balanceThreshold;
        pdqsort(mid + 1, b, limit);
        b = mid;
      }
    }
  }
};
using WarpSorter = WarpSorterT<int>;
