// vb_diff.h -- the order-preserving matching of a recompose (vb_recompose, vb_compose.cu): which instances of the old composition
// reappear, unchanged, in the new one. Plain C++, no CUDA.
//
// match[j] = i pairs new element j with old element i (VB_DIFF_NONE: unpaired). Pairs are between equal elements only, and
// i < i' whenever j < j': any such matching is sound for damage; a longer one only damages less. The common prefix and suffix
// are paired first; Myers' O((N + M) D) greedy diff pairs a longest common subsequence of the middle when the middle needs at
// most VB_RECOMPOSE_MAX_EDITS insertions and deletions; past that, the middle is paired by position where the elements are equal.
// The cost stays O(N + M) with a constant factor of VB_RECOMPOSE_MAX_EDITS.
#ifndef VB_DIFF_H
#define VB_DIFF_H
#include <stdint.h>

#include <vector>

#include "../../include/vello_b200.h"

#define VB_DIFF_NONE 0xffffffffu

// eq(i, j): old element i equals new element j. Returns the edit count of the middle, or VB_RECOMPOSE_MAX_EDITS + 1 when it was
// paired by position.
template <class Eq> static uint32_t vb_diff_match(uint32_t n_old, uint32_t n_new, Eq eq, uint32_t *match) {
    for (uint32_t j = 0; j < n_new; j++) match[j] = VB_DIFF_NONE;
    uint32_t pre = 0, suf = 0;
    while (pre < n_old && pre < n_new && eq(pre, pre)) {
        match[pre] = pre;
        pre++;
    }
    while (suf < n_old - pre && suf < n_new - pre && eq(n_old - 1u - suf, n_new - 1u - suf)) {
        match[n_new - 1u - suf] = n_old - 1u - suf;
        suf++;
    }
    // the middle: old [pre, pre + N), new [pre, pre + M)
    const int N = (int)(n_old - pre - suf), M = (int)(n_new - pre - suf), D_MAX = (int)VB_RECOMPOSE_MAX_EDITS;
    if (N == 0 || M == 0) return (uint32_t)(N + M);
    auto same = [&](int x, int y) { return eq(pre + (uint32_t)x, pre + (uint32_t)y); };
    // V[k + off]: the furthest x on diagonal k = x - y after d edits; trace[d] holds V before step d
    const int off = D_MAX + 1;
    std::vector<int> V(2 * D_MAX + 3, 0);
    std::vector<std::vector<int>> trace;
    int D = -1;
    for (int d = 0; d <= D_MAX && D < 0; d++) {
        trace.push_back(V);
        for (int k = -d; k <= d; k += 2) {
            int x = (k == -d || (k != d && V[off + k - 1] < V[off + k + 1])) ? V[off + k + 1] : V[off + k - 1] + 1;
            int y = x - k;
            while (x < N && y < M && same(x, y)) x++, y++;
            V[off + k] = x;
            if (x >= N && y >= M) {
                D = d;
                break;
            }
        }
    }
    if (D < 0) { // too many edits: by position
        for (int x = 0; x < N && x < M; x++)
            if (same(x, x)) match[pre + (uint32_t)x] = pre + (uint32_t)x;
        return VB_RECOMPOSE_MAX_EDITS + 1u;
    }
    // back from (N, M): each step's snake is a run of pairs
    int x = N, y = M;
    for (int d = D; d >= 0; d--) {
        const std::vector<int> &P = trace[(size_t)d];
        const int k = x - y;
        const int pk = (k == -d || (k != d && P[off + k - 1] < P[off + k + 1])) ? k + 1 : k - 1;
        const int px = d == 0 ? 0 : P[off + pk], py = d == 0 ? 0 : px - pk;
        const int sx = d == 0 ? 0 : (pk == k + 1 ? px : px + 1); // where the snake starts, after step d's edit
        for (; x > sx && y > sx - k; x--, y--) match[pre + (uint32_t)(y - 1)] = pre + (uint32_t)(x - 1);
        x = px;
        y = py;
    }
    return (uint32_t)D;
}

#endif
