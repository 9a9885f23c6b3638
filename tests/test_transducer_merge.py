"""CPU check of the transducer search's arg-max / log-sum-exp merge (speechbrain_b200/csrc/transducer_merge.cuh, the
host- and device-callable functions the search kernel uses) on rows with NaN, +inf and -inf logits.

A small C++ driver, built here with the host compiler, splits each row into contiguous per-CTA slices as the kernel does,
scans every slice, folds the partials in three different orders and prints the decision.  It must be the reference's
decision -- torch.max over log_softmax(logits), which is what TransducerBeamSearcher.transducer_greedy_decode takes -- for
every order, and always a valid vocabulary index (the search uses the token to index its input table)."""
import os
import shutil
import subprocess

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

DRIVER = r"""
#include <cstdio>
#include <vector>
#include "transducer_merge.cuh"
using namespace sbk::td;
int main() {
    int n, V, G;
    if (scanf("%d", &n) != 1) return 1;
    for (int r = 0; r < n; ++r) {
        if (scanf("%d %d", &V, &G) != 2) return 1;
        std::vector<float> x(V);
        for (int v = 0; v < V; ++v) { double d; if (scanf("%lf", &d) != 1) return 1; x[v] = (float)d; }
        const int nv = (V + G - 1) / G;
        std::vector<float> pm(G), ps(G);
        std::vector<int> pa(G);
        for (int g = 0; g < G; ++g) {   // one CTA's slice: scan, then the sum of exp(x - max)
            const int v0 = g * nv < V ? g * nv : V, v1 = v0 + nv < V ? v0 + nv : V;
            float m = -INFINITY; int a = NO_ARG;
            for (int v = v1 - 1; v >= v0; --v)   // reverse scan: the order must not matter
                if (argmax_before(x[v], v, m, a)) { m = x[v]; a = v; }
            float s = 0.f;
            for (int v = v0; v < v1; ++v) s += expf(x[v] - m);
            pm[g] = m; pa[g] = a; ps[g] = s;
        }
        int out[3];
        for (int order = 0; order < 3; ++order) {
            float m = -INFINITY, s = 0.f; int a = NO_ARG;
            for (int k = 0; k < G; ++k) {
                const int g = order == 0 ? k : order == 1 ? G - 1 - k : (k * 7) % G;
                lse_merge(m, a, s, pm[g], pa[g], ps[g]);
            }
            out[order] = decision(m, a, V);
        }
        printf("%d %d %d\n", out[0], out[1], out[2]);
    }
    return 0;
}
"""


def _compiler():
    for c in ("g++", "c++", "clang++"):
        if shutil.which(c):
            return c
    pytest.skip("no host C++ compiler")


def _rows():
    g = torch.Generator().manual_seed(0)
    nan, inf = float("nan"), float("inf")
    rows = []
    for V in (7, 512, 1000):
        base = torch.randn(V, generator=g) * 3
        rows.append(base.clone())                                  # finite
        r = base.clone(); r[V // 3] = nan; rows.append(r)          # one NaN
        r = base.clone(); r[V // 2] = nan; r[V - 1] = nan; rows.append(r)
        rows.append(torch.full((V,), nan))                         # all NaN
        r = base.clone(); r[V // 4] = inf; r[V - 2] = inf; rows.append(r)   # +inf, twice
        rows.append(torch.full((V,), -inf))                        # all -inf
        r = torch.full((V,), -inf); r[V - 1] = 2.0; rows.append(r)  # one finite among -inf
        r = base.clone(); r[1] = -inf; r[V - 1] = inf; r[3 % V] = nan; rows.append(r)
    return rows


def test_merge_matches_reference_decision_on_non_finite_logits(tmp_path):
    src = tmp_path / "merge.cpp"
    src.write_text(DRIVER)
    exe = tmp_path / "merge"
    subprocess.run([_compiler(), "-std=c++17", "-O1", "-I", os.path.join(ROOT, "speechbrain_b200", "csrc"), str(src), "-o",
                    str(exe)], check=True)
    cases = [(r, G) for r in _rows() for G in (1, 5, 132)]
    lines = [str(len(cases))]
    for r, G in cases:
        lines.append(f"{r.numel()} {G} " + " ".join(repr(float(v)) for v in r.tolist()))
    out = subprocess.run([str(exe)], input="\n".join(lines), capture_output=True, text=True, check=True).stdout.split("\n")
    for (r, G), line in zip(cases, out):
        got = [int(x) for x in line.split()]
        ref = int(torch.max(torch.log_softmax(r, dim=-1), dim=-1).indices)
        assert got == [ref] * 3, (r.numel(), G, got, ref)
        assert 0 <= ref < r.numel()
