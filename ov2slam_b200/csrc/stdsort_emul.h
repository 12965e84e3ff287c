// Restatement of libstdc++'s std::sort (introsort: median-of-3 quicksort to partitions of <= 16,
// heapsort when the depth limit 2*floor(log2 n) is hit, then a final insertion sort), for the one
// use the reference makes of it: std::sort(vkps.begin(), vkps.end(), compare_response) with
// compare_response(a, b) = a.response > b.response (/root/reference/src/feature_extractor.cpp:75-77,
// :518), after which only element 0 is read (:521).  std::sort is not stable, so when several
// keypoints share the maximal response the winner is decided by this exact sequence of
// comparisons and swaps - which is what must be reproduced for bit-exact keypoints.
//
// Keys are (response, original index) pairs packed in one int: key = (response << 16) | index
// (response <= 254, index < 65536: a cell holds at most a few thousand candidates),
// compared on the response part only.  Compiles for host (unit-tested against the real
// std::sort in tests/test_stdsort_emul.py) and device (used by the grid-FAST sweep).
#pragma once

#ifdef __CUDACC__
#define OV2_HD __host__ __device__ __forceinline__
#else
#define OV2_HD static inline
#endif

namespace ov2sort {

// comp(a, b) == compare_response(a, b): strictly greater response
OV2_HD bool gt(int a, int b) { return (a >> 16) > (b >> 16); }
OV2_HD void swp(int* v, int i, int j) { int t = v[i]; v[i] = v[j]; v[j] = t; }

OV2_HD void move_median_to_first(int* v, int result, int a, int b, int c) {
    if (gt(v[a], v[b])) {
        if (gt(v[b], v[c])) swp(v, result, b);
        else if (gt(v[a], v[c])) swp(v, result, c);
        else swp(v, result, a);
    } else if (gt(v[a], v[c])) swp(v, result, a);
    else if (gt(v[b], v[c])) swp(v, result, c);
    else swp(v, result, b);
}

OV2_HD int unguarded_partition(int* v, int first, int last, int pivot) {
    for (;;) {
        while (gt(v[first], v[pivot])) ++first;
        --last;
        while (gt(v[pivot], v[last])) --last;
        if (!(first < last)) return first;
        swp(v, first, last);
        ++first;
    }
}

OV2_HD void push_heap_(int* v, int first, int hole, int top, int value) {
    int parent = (hole - 1) / 2;
    while (hole > top && gt(v[first + parent], value)) {
        v[first + hole] = v[first + parent];
        hole = parent;
        parent = (hole - 1) / 2;
    }
    v[first + hole] = value;
}

OV2_HD void adjust_heap(int* v, int first, int hole, int len, int value) {
    const int top = hole;
    int child = hole;
    while (child < (len - 1) / 2) {
        child = 2 * (child + 1);
        if (gt(v[first + child], v[first + (child - 1)])) child--;
        v[first + hole] = v[first + child];
        hole = child;
    }
    if ((len & 1) == 0 && child == (len - 2) / 2) {
        child = 2 * (child + 1);
        v[first + hole] = v[first + (child - 1)];
        hole = child - 1;
    }
    push_heap_(v, first, hole, top, value);
}

// std::__partial_sort(first, last, last) == make_heap + sort_heap on [first, last)
OV2_HD void heap_sort(int* v, int first, int last) {
    const int len = last - first;
    if (len >= 2) {
        int parent = (len - 2) / 2;
        for (;;) {
            int value = v[first + parent];
            adjust_heap(v, first, parent, len, value);
            if (parent == 0) break;
            parent--;
        }
    }
    int l = last;
    while (l - first > 1) {
        --l;
        int value = v[l];
        v[l] = v[first];
        adjust_heap(v, first, 0, l - first, value);
    }
}

OV2_HD void insertion_sort(int* v, int first, int last) {
    if (first == last) return;
    for (int i = first + 1; i != last; ++i) {
        int val = v[i];
        if (gt(val, v[first])) {
            for (int k = i; k > first; --k) v[k] = v[k - 1];
            v[first] = val;
        } else {
            int k = i;
            while (gt(val, v[k - 1])) { v[k] = v[k - 1]; --k; }
            v[k] = val;
        }
    }
}

OV2_HD void unguarded_insertion_sort(int* v, int first, int last) {
    for (int i = first; i != last; ++i) {
        int val = v[i];
        int k = i;
        while (gt(val, v[k - 1])) { v[k] = v[k - 1]; --k; }
        v[k] = val;
    }
}

// In-place std::sort of v[0..n) (the explicit stack replaces the recursion of __introsort_loop,
// which recurses on the right part and iterates on the left; it holds at most 2 log2(n) ranges).
OV2_HD void sort_desc(int* v, int n) {
    if (n < 2) return;
    int lg = 0;
    for (int t = n; t > 1; t >>= 1) ++lg;
    int stack_first[40], stack_last[40], stack_depth[40];
    int sp = 0;
    stack_first[0] = 0; stack_last[0] = n; stack_depth[0] = 2 * lg; sp = 1;
    while (sp > 0) {
        --sp;
        int first = stack_first[sp], last = stack_last[sp], depth = stack_depth[sp];
        // __introsort_loop(first, last, depth): recursion order is (cut,last) first, then the
        // loop continues on (first,cut).  The two sub-ranges are disjoint, so the order in which
        // they are processed does not change the result; process left iteratively, push right.
        while (last - first > 16) {
            if (depth == 0) { heap_sort(v, first, last); break; }
            --depth;
            int mid = first + (last - first) / 2;
            move_median_to_first(v, first, first + 1, mid, last - 1);
            int cut = unguarded_partition(v, first + 1, last, first);
            stack_first[sp] = cut; stack_last[sp] = last; stack_depth[sp] = depth; ++sp;
            last = cut;
        }
    }
    if (n > 16) {
        insertion_sort(v, 0, 16);
        unguarded_insertion_sort(v, 16, n);
    } else {
        insertion_sort(v, 0, n);
    }
}

// The element sort_desc(v, n) leaves at v[0], for a caller that reads nothing else (the reference reads only
// vkps.at(0)).  __introsort_loop's recursion into (cut, last) never touches [first, cut), and every element right of a
// cut has a response no larger than every element left of it, so the final insertion sort cannot move one of them in
// front of the leftmost partition: only the leftmost chain of partitions has to be followed, n + n/2 + ... steps
// instead of the whole sort.  v is left permuted but not sorted.
OV2_HD int sort_desc_front(int* v, int n) {
    if (n < 2) return v[0];
    int lg = 0;
    for (int t = n; t > 1; t >>= 1) ++lg;
    int last = n, depth = 2 * lg;
    while (last > 16) {
        if (depth == 0) { heap_sort(v, 0, last); break; }
        --depth;
        move_median_to_first(v, 0, 1, last / 2, last - 1);
        last = unguarded_partition(v, 1, last, 0);
    }
    insertion_sort(v, 0, last < 16 ? last : 16);
    return v[0];
}

}  // namespace ov2sort
