// TEST INFRASTRUCTURE -- CPU oracle (see orc_requirement.hpp header).
//
// orc_gosort.hpp: restatement of Go's sort.Slice, i.e. pdqsort_func of the Go standard library (package sort,
// zsortfunc.go, go1.19+ .. go1.26: pattern-defeating quicksort).  The reference calls sort.Slice at
//   scheduler.go:504 (newNodeClaims by len(Pods)), queue.go:38, cloudprovider/types.go:240 (OrderByPrice),
//   disruption/consolidation.go:127 (sortCandidates)
// and the permutation it leaves among EQUAL keys decides which NodeClaim a pod lands on (SURVEY.md H2).
// The Go standard library is not part of the reference repository (third-party: Go toolchain go1.26.3 per go.mod), so this
// follows the published algorithm; tie-order parity against a real Go run is UNPINNED (no reference test asserts it).
#pragma once
#include <cstdint>

namespace orc {

// data.Less(i,j) / data.Swap(i,j) over indices, like sort's lessSwap
template <class LessFn, class SwapFn>
struct GoSorter {
  LessFn less;
  SwapFn swap;
  GoSorter(LessFn l, SwapFn s) : less(l), swap(s) {}

  enum Hint { unknownHint = 0, increasingHint = 1, decreasingHint = 2 };

  static int bits_len(uint64_t x) {
    int n = 0;
    while (x) {
      n++;
      x >>= 1;
    }
    return n;
  }

  void insertion_sort(int a, int b) {
    for (int i = a + 1; i < b; i++)
      for (int j = i; j > a && less(j, j - 1); j--) swap(j, j - 1);
  }
  void sift_down(int lo, int hi, int first) {
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
  void heap_sort(int a, int b) {
    int first = a, lo = 0, hi = b - a;
    for (int i = (hi - 1) / 2; i >= 0; i--) sift_down(i, hi, first);
    for (int i = hi - 1; i >= 0; i--) {
      swap(first, first + i);
      sift_down(lo, i, first);
    }
  }
  // partition_func: returns new pivot index, sets already_partitioned
  int partition(int a, int b, int pivot, bool* already) {
    swap(a, pivot);
    int i = a + 1, j = b - 1;
    while (i <= j && less(i, a)) i++;
    while (i <= j && !less(j, a)) j--;
    if (i > j) {
      swap(j, a);
      *already = true;
      return j;
    }
    swap(i, j);
    i++;
    j--;
    for (;;) {
      while (i <= j && less(i, a)) i++;
      while (i <= j && !less(j, a)) j--;
      if (i > j) break;
      swap(i, j);
      i++;
      j--;
    }
    swap(j, a);
    *already = false;
    return j;
  }
  int partition_equal(int a, int b, int pivot) {
    swap(a, pivot);
    int i = a + 1, j = b - 1;
    for (;;) {
      while (i <= j && !less(a, i)) i++;
      while (i <= j && less(a, j)) j--;
      if (i > j) break;
      swap(i, j);
      i++;
      j--;
    }
    return i;
  }
  bool partial_insertion_sort(int a, int b) {
    const int maxSteps = 5, shortestShifting = 50;
    int i = a + 1;
    for (int j = 0; j < maxSteps; j++) {
      while (i < b && !less(i, i - 1)) i++;
      if (i == b) return true;
      if (b - a < shortestShifting) return false;
      swap(i, i - 1);
      if (i - a >= 2) {
        for (int k = i - 1; k >= 1; k--) {
          if (!less(k, k - 1)) break;
          swap(k, k - 1);
        }
      }
      if (b - i >= 2) {
        for (int k = i + 1; k < b; k++) {
          if (!less(k, k - 1)) break;
          swap(k, k - 1);
        }
      }
    }
    return false;
  }
  static uint64_t xorshift_next(uint64_t* r) {
    *r ^= *r << 13;
    *r ^= *r >> 7;
    *r ^= *r << 17;
    return *r;
  }
  void break_patterns(int a, int b) {
    int length = b - a;
    if (length >= 8) {
      uint64_t random = (uint64_t)length;
      uint64_t modulus = 1ull << bits_len((uint64_t)length);
      int idx = a + (length / 4) * 2 - 1;
      for (int i = 0; i < 3; i++) {
        int other = (int)(xorshift_next(&random) & (modulus - 1));
        if (other >= length) other -= length;
        swap(idx - 1 + i, a + other);
      }
    }
  }
  void order2(int* a, int* b, int* swaps) {
    if (less(*b, *a)) {
      (*swaps)++;
      int t = *a;
      *a = *b;
      *b = t;
    }
  }
  int median(int a, int b, int c, int* swaps) {
    order2(&a, &b, swaps);
    order2(&b, &c, swaps);
    order2(&a, &b, swaps);
    return b;
  }
  int median_adjacent(int a, int* swaps) { return median(a - 1, a, a + 1, swaps); }
  int choose_pivot(int a, int b, Hint* hint) {
    const int shortestNinther = 50, maxSwaps = 4 * 3;
    int l = b - a;
    int swaps = 0;
    int i = a + l / 4 * 1, j = a + l / 4 * 2, k = a + l / 4 * 3;
    if (l >= 8) {
      if (l >= shortestNinther) {
        i = median_adjacent(i, &swaps);
        j = median_adjacent(j, &swaps);
        k = median_adjacent(k, &swaps);
      }
      j = median(i, j, k, &swaps);
    }
    if (swaps == 0)
      *hint = increasingHint;
    else if (swaps == maxSwaps)
      *hint = decreasingHint;
    else
      *hint = unknownHint;
    return j;
  }
  void reverse_range(int a, int b) {
    int i = a, j = b - 1;
    while (i < j) {
      swap(i, j);
      i++;
      j--;
    }
  }
  void pdqsort(int a, int b, int limit) {
    const int maxInsertion = 12;
    bool wasBalanced = true, wasPartitioned = true;
    for (;;) {
      int length = b - a;
      if (length <= maxInsertion) {
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
      Hint hint;
      int pivot = choose_pivot(a, b, &hint);
      if (hint == decreasingHint) {
        reverse_range(a, b);
        pivot = (b - 1) - (pivot - a);
        hint = increasingHint;
      }
      if (wasBalanced && wasPartitioned && hint == increasingHint) {
        if (partial_insertion_sort(a, b)) return;
      }
      if (a > 0 && !less(a - 1, pivot)) {
        int mid = partition_equal(a, b, pivot);
        a = mid;
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
  // sort.Slice(x, less): n := len; limit := bits.Len(uint(n)); pdqsort_func(data, 0, n, limit)
  void sort(int n) { pdqsort(0, n, bits_len((uint64_t)n)); }
};

template <class LessFn, class SwapFn>
inline void go_sort_slice(int n, LessFn less, SwapFn swap) {
  GoSorter<LessFn, SwapFn> s(less, swap);
  s.sort(n);
}

// sort.SliceStable == insertion-sorted blocks of 20 + symMerge; any stable algorithm gives the same permutation.

}  // namespace orc
