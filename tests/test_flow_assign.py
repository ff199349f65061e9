"""The association programme of samples of K > 2 frames (reference solvers.py:9-138 for any len(det_split)) as a
min-cost flow: csrc/flow_assign.cu through mmmot_b200.solve_frames / ortools_solve / TrackingModule.predict.

CPU: the MILP restatement (oracle/lp_ref.py) is pinned for K > 2 by exhaustive enumeration, a numpy restatement of the
kernel's algorithm (same network, potentials and tie rules) agrees with it, and the C ABI rejects bad arguments before
any CUDA call.  GPU: the kernel against the MILP restatement, bit for bit on unique optima."""
import copy
import ctypes
import itertools

import numpy as np
import pytest
import torch

from oracle import lp_ref

S_NODE, T_NODE = 0, 1
NONE, NEW, END = -1, -2, -2


def _rand_frames(g, counts, B=1, scale=None):
    """Random scores of B samples in the forward's layout: det / new / end B x L (new zero on frame 0, end zero on the
    last frame), links K - 1 tensors B x n_i x n_{i+1}.  Continuous (unique optimum), or integers in [-scale, scale]."""
    L = sum(counts)

    def draw(*shape):
        if scale is None:
            return torch.rand(*shape, generator=g)
        return torch.randint(-scale, scale + 1, shape, generator=g).float()
    if scale is None:
        det = draw(B, L) - (draw(B, L) < 0.3).float()
        links = [draw(B, a, b) - 0.25 for a, b in zip(counts[:-1], counts[1:])]
        new, end = draw(B, L) - 0.2, draw(B, L) - 0.2
    else:
        det, new, end = draw(B, L), draw(B, L), draw(B, L)
        links = [draw(B, a, b) for a, b in zip(counts[:-1], counts[1:])]
    new[:, :counts[0]] = 0
    end[:, L - counts[-1]:] = 0
    return det, links, new, end


def _milp(det, links, new, end, counts, b=0, exclude=None):
    return lp_ref.milp_solve(det[b], [l[b:b + 1] for l in links], new[b], end[b], counts, exclude=exclude)


def _same(got, ref):
    return (torch.equal(got[0], ref[0]) and len(got[1]) == len(ref[1]) and all(torch.equal(a, b) for a, b in zip(got[1], ref[1]))
            and torch.equal(got[2], ref[2]) and torch.equal(got[3], ref[3]))


def _objective(det, links, new, end, a):
    """Reference objective (solvers.py:31-49) in fp64 of an assignment tuple."""
    v = (det.double() * a[0].double()).sum() + (new.double() * a[2].double()).sum() + (end.double() * a[3].double()).sum()
    return float(v + sum((l.double() * x.double()).sum() for l, x in zip(links, a[1])))


def _feasible(a, counts):
    """The flow constraints of solvers.py:83-111 on an assignment tuple (0/1 tensors)."""
    ad, al, an, ae = a[0].double(), [x[0].double() for x in a[1]], a[2].double(), a[3].double()
    off = np.concatenate([[0], np.cumsum(counts)])
    for t in (ad, an, ae, *al):
        if not bool(((t == 0) | (t == 1)).all()):
            return False
    for f in range(len(counts)):
        s = slice(int(off[f]), int(off[f + 1]))
        succ = al[f].sum(1) if f + 1 < len(counts) else torch.zeros(counts[f], dtype=torch.float64)
        pred = al[f - 1].sum(0) if f > 0 else torch.zeros(counts[f], dtype=torch.float64)
        if not (torch.equal(ae[s] + succ, ad[s]) and torch.equal(an[s] + pred, ad[s])):
            return False
    return True


# ------------------------------------------------------------------ exhaustive enumeration (tiny K-frame samples)
def _partial_matchings(n, m):
    """Every injective partial map from n detections to m (entry -1 = no successor)."""
    for mt in itertools.product(range(-1, m), repeat=n):
        used = [k for k in mt if k >= 0]
        if len(used) == len(set(used)):
            yield mt


def _enumerate(det, links, new, end, counts):
    """Best and second-best 0/1 solution of the programme: enumerate the det flags and a partial matching per
    transition, derive new = det - predecessors and end = det - successors from the equalities of solvers.py:83-111,
    keep the solutions whose new and end are 0/1.  Returns (assignment tuple, best objective, second-best objective)."""
    K, L = len(counts), sum(counts)
    off = np.concatenate([[0], np.cumsum(counts)])
    d, nw, e = (np.asarray(t, np.float64).reshape(-1) for t in (det, new, end))
    lk = [np.asarray(l, np.float64).reshape(a, b) for l, a, b in zip(links, counts[:-1], counts[1:])]
    flags = np.array(list(itertools.product((0, 1), repeat=L)), np.float64)        # every det flag vector at once
    best, second, best_sol = -np.inf, -np.inf, None
    for mts in itertools.product(*[list(_partial_matchings(a, b)) for a, b in zip(counts[:-1], counts[1:])]):
        succ, pred, lsum = np.zeros(L), np.zeros(L), 0.0
        for f, mt in enumerate(mts):
            for j, k in enumerate(mt):
                if k >= 0:
                    succ[off[f] + j] += 1
                    pred[off[f + 1] + k] += 1
                    lsum += lk[f][j, k]
        a_new, a_end = flags - pred, flags - succ
        ok = ((a_new == 0) | (a_new == 1)).all(1) & ((a_end == 0) | (a_end == 1)).all(1)
        if not ok.any():
            continue
        obj = flags @ d + a_new @ nw + a_end @ e + lsum
        obj = np.where(ok, obj, -np.inf)
        for r in np.argsort(-obj)[:2]:
            if not ok[r]:
                continue
            if obj[r] > best:
                second, best = best, obj[r]
                al = [np.zeros((a, b)) for a, b in zip(counts[:-1], counts[1:])]
                for f, mt in enumerate(mts):
                    for j, k in enumerate(mt):
                        if k >= 0:
                            al[f][j, k] = 1
                best_sol = (flags[r], al, a_new[r], a_end[r])
            elif obj[r] > second:
                second = obj[r]
    t = lambda a: torch.as_tensor(a, dtype=torch.float32)
    fd, al, fn, fe = best_sol
    return (t(fd), [t(x[None]) for x in al], t(fn), t(fe)), float(best), float(second)


@pytest.mark.parametrize("counts", [(3, 3, 3), (2, 1, 3), (1, 4, 2), (2, 3, 2, 2), (1, 2, 2, 1), (3, 1, 1, 2)])
def test_milp_restatement_matches_enumeration_k_frames(counts):
    """lp_ref.milp_solve builds the K-frame model (its _build loops over det_split); exhaustive enumeration of the
    0/1 solutions pins it for K = 3 and 4."""
    g = torch.Generator().manual_seed(sum(c * 7 ** i for i, c in enumerate(counts)))
    for _ in range(3):
        det, links, new, end = _rand_frames(g, list(counts))
        (a, obj, _) = _milp(det, links, new, end, list(counts))
        b, best, second = _enumerate(det[0], [l[0] for l in links], new[0], end[0], list(counts))
        assert abs(obj - best) < 1e-9
        assert best - second > 1e-6
        assert _same(a, b)


# ------------------------------------------------------------------ numpy restatement of csrc/flow_assign.cu
def flow_rehearsal(det, links, new, end, counts):
    """The kernel's algorithm on one sample, node for node: S = 0, T = 1, in_d = 2 + 2d, out_d = 3 + 2d; initial
    potentials by a frame-by-frame sweep of the acyclic network; per augmentation a dense Dijkstra on reduced costs
    (clamped at 0) that settles the smallest (distance, node) first and stops at T, potentials moved by
    min(d(v), d(T)), and the path augmented only when the new pi(T) (its cost) is < 0.  Scores are read from fp32."""
    K, L = len(counts), sum(counts)
    V = 2 * L + 2
    off = np.concatenate([[0], np.cumsum(counts)]).astype(int)
    fr = np.repeat(np.arange(K), counts)
    d, nw, e = (np.asarray(t, np.float32).astype(np.float64).reshape(-1) for t in (det, new, end))
    lk = [np.asarray(l, np.float32).astype(np.float64).reshape(a, b) for l, a, b in zip(links, counts[:-1], counts[1:])]
    IN = lambda i: 2 + 2 * np.asarray(i)
    OUT = lambda i: 3 + 2 * np.asarray(i)
    pred, succ, on = np.full(L, NONE), np.full(L, NONE), np.zeros(L, bool)
    pi = np.zeros(V)
    for f in range(K):
        o, nf = off[f], counts[f]
        m = -nw[o:o + nf]
        if f > 0:
            m = np.minimum(m, (pi[OUT(np.arange(off[f - 1], o))][:, None] - lk[f - 1]).min(0))
        pi[IN(np.arange(o, o + nf))] = m
        pi[OUT(np.arange(o, o + nf))] = m - d[o:o + nf]
    pi[T_NODE] = (pi[OUT(np.arange(L))] - e).min()
    for _ in range(L):
        dist, par, settled = np.full(V, np.inf), np.full(V, -1), np.zeros(V, bool)
        dist[S_NODE] = 0.0
        reached = False
        for _ in range(V):
            cand = np.where(settled, np.inf, dist)
            u = int(np.argmin(cand))                  # first minimum: the smaller node index wins a tie
            if not cand[u] < np.inf:
                break
            du = cand[u]
            settled[u] = True
            if u == T_NODE:
                reached = True
                break
            vs, cs = [], []
            if u == S_NODE:
                i = np.flatnonzero(pred != NEW)
                vs, cs = IN(i), -nw[i]
            elif u % 2 == 0:
                i = (u - 2) // 2
                if not on[i]:
                    vs, cs = [OUT(i)], [-d[i]]
                elif pred[i] >= 0:
                    f = fr[i]
                    vs, cs = [OUT(off[f - 1] + pred[i])], [lk[f - 1][pred[i], i - off[f]]]
            else:
                i = (u - 3) // 2
                f = fr[i]
                if succ[i] != END:
                    vs.append(T_NODE); cs.append(-e[i])
                if on[i]:
                    vs.append(IN(i)); cs.append(d[i])
                if f + 1 < K:
                    k = np.flatnonzero(np.arange(counts[f + 1]) != succ[i])
                    vs = np.concatenate([np.asarray(vs, int), IN(off[f + 1] + k)])
                    cs = np.concatenate([np.asarray(cs, float), -lk[f][i - off[f], k]])
            vs, cs = np.asarray(vs, int).reshape(-1), np.asarray(cs, float).reshape(-1)
            if vs.size:
                nd = du + np.maximum(cs + pi[u] - pi[vs], 0.0)
                better = ~settled[vs] & (nd < dist[vs])
                dist[vs[better]] = nd[better]
                par[vs[better]] = u
        if not reached:
            break
        pi += np.minimum(dist, dist[T_NODE])
        if not pi[T_NODE] < 0.0:
            break
        v = T_NODE
        for _ in range(V):
            if v == S_NODE:
                break
            p = par[v]
            if p == S_NODE:
                pred[(v - 2) // 2] = NEW
            elif v == T_NODE:
                succ[(p - 2) // 2] = END
            else:
                a, b = (p - 2) // 2, (v - 2) // 2
                la, lb = a - off[fr[a]], b - off[fr[b]]
                if a == b:
                    on[a] = p % 2 == 0
                elif p % 2:
                    succ[a], pred[b] = lb, la
                else:
                    if succ[b] == la:
                        succ[b] = NONE
                    if pred[a] == lb:
                        pred[a] = NONE
            v = p
    al = [np.zeros((a, b), np.float32) for a, b in zip(counts[:-1], counts[1:])]
    for i in range(L - counts[-1]):
        if succ[i] >= 0:
            al[fr[i]][i - off[fr[i]], succ[i]] = 1
    t = lambda a: torch.as_tensor(np.asarray(a, np.float32))
    return t(on), [t(x[None]) for x in al], t(pred == NEW), t(succ == END)


@pytest.mark.parametrize("K,n", [(2, 6), (3, 4), (3, 12), (4, 8), (5, 16), (5, 32)])
def test_flow_rehearsal_matches_milp(K, n):
    """The kernel's algorithm, restated in numpy with the same arcs, potentials and tie rules, returns the MILP's
    0/1 solution on random continuous scores (ragged counts, one-detection frames included)."""
    g = torch.Generator().manual_seed(1000 * K + n)
    for _ in range(3 if n <= 16 else 1):
        counts = [int(c) for c in torch.randint(1, n + 1, (K,), generator=g)]
        counts[int(torch.randint(0, K, (1,), generator=g))] = n
        det, links, new, end = _rand_frames(g, counts)
        (a, obj, _) = _milp(det, links, new, end, counts)
        got = flow_rehearsal(det[0], [l[0] for l in links], new[0], end[0], counts)
        assert _same(got, a), counts
        assert abs(_objective(det[0], [l[:1] for l in links], new[0], end[0], got) - obj) < 1e-9


def test_flow_rehearsal_on_ties_is_optimal():
    """Integer scores (many optima): the restated algorithm still returns a feasible optimum."""
    g = torch.Generator().manual_seed(3)
    for counts in ([3, 5, 2], [4, 4, 4, 4], [1, 6, 6, 1, 3]):
        det, links, new, end = _rand_frames(g, counts, scale=2)
        (_, obj, _) = _milp(det, links, new, end, counts)
        got = flow_rehearsal(det[0], [l[0] for l in links], new[0], end[0], counts)
        assert _feasible(got, counts)
        assert abs(_objective(det[0], [l[:1] for l in links], new[0], end[0], got) - obj) < 1e-9


# ------------------------------------------------------------------ C ABI / Python surface without a GPU
def test_flow_abi_rejects_bad_arguments(lib_built):
    from mmmot_b200 import _lib
    lib = _lib.load()
    p = ctypes.c_void_p(256)                   # never dereferenced: every case below is refused before any CUDA call

    def call(counts, frames=None, samples=1, null=None):
        c = (ctypes.c_int * max(len(counts), 1))(*counts)
        ptrs = [p] * 9
        if null is not None:
            ptrs[null] = None
        det, links, new, end, ad, al, an, ae, mt = ptrs
        return lib.mmmot_flow_assign(det, 0, links, 0, new, 0, end, 0, samples, len(counts) if frames is None else frames,
                                     c, ad, al, an, ae, mt, p, 256, None)
    for k in range(9):
        assert call([3, 4, 5], null=k) == -1, k
    assert lib.mmmot_flow_assign(p, 0, p, 0, p, 0, p, 0, 1, 3, None, p, p, p, p, p, p, 256, None) == -1   # counts
    assert call([3]) == -1                                  # frames < 2
    assert call([3, 4], frames=0) == -1
    assert call([3, 4], samples=0) == -1
    assert call([3, 0, 5]) == -1                            # a zero count
    assert call([3, -2, 5]) == -1
    assert call([1] * 65) == -3                             # above the frame cap
    assert call([2235, 2235]) == -3                         # L = 4470: one sample's state exceeds shared memory
    assert call([1500, 1500, 1470]) == -3
    assert call([1] * 64 + [0]) == -1                       # a bad count is an argument error whatever the shape
    assert call([2235, 2235, -1]) == -1
    assert lib.mmmot_flow_workspace(4, 3, (ctypes.c_int * 3)(3, 4, 5)) > 0


def test_ortools_solve_link_count_mismatch():
    import mmmot_b200
    z = torch.zeros
    with pytest.raises(ValueError):
        mmmot_b200.ortools_solve(z(9), [z(1, 3, 3)], z(9), z(9), [3, 3, 3])
    with pytest.raises(ValueError):
        mmmot_b200.ortools_solve(z(6), [z(1, 3, 3), z(1, 3, 3)], z(6), z(6), [3, 3])
    with pytest.raises(NotImplementedError):
        mmmot_b200.ortools_solve(z(9), [z(1, 3, 3)] * 2, z(9), z(9), [3, 3, 3], gt=object())


# ------------------------------------------------------------------ GPU
def _gpu_rows(r, b):
    return (r["assign_det"][b].cpu(), [x[b:b + 1].cpu() for x in r["assign_link"]], r["assign_new"][b].cpu(),
            r["assign_end"][b].cpu())


def _frame_cap_counts():
    g = torch.Generator().manual_seed(64)
    return tuple(int(c) for c in torch.randint(1, 5, (64,), generator=g))


@pytest.mark.gpu
@pytest.mark.parametrize("counts,B,gap", [
    ((5, 1, 7), 4, True), ((3, 1, 4, 2), 4, True), ((6, 1, 5, 8, 1, 4), 3, True), ((9, 4, 1, 12, 7, 3, 1, 10), 3, True),
    ((32, 1, 32), 2, False), ((128, 97, 128), 2, False), ((40, 64, 1, 64, 33, 64), 2, False),
    (_frame_cap_counts(), 2, False)])
def test_flow_bit_exact_vs_milp(counts, B, gap):
    """B samples per call read through strided views of forward-shaped outputs (det B x 3 x L, links B x 3 x n x m,
    the test_mode stack 2 selected): the 0/1 tensors equal the MILP's on random continuous scores, match agrees with
    assign_link, and, where `gap`, the second-best solution is strictly worse."""
    import mmmot_b200
    counts = list(counts)
    L = sum(counts)
    g = torch.Generator().manual_seed(sum(counts) * len(counts))
    det, links, new, end = _rand_frames(g, counts, B)
    stack = lambda t: torch.stack([torch.rand_like(t), torch.rand_like(t), t], 1).cuda()
    sdet, snew, send = stack(det), stack(new), stack(end)
    slinks = [stack(l) for l in links]
    r = mmmot_b200.solve_frames(sdet[:, 2], [l[:, 2] for l in slinks], snew[:, 2], send[:, 2], counts)
    assert r["match"].shape == (B, L - counts[-1]) and [tuple(x.shape) for x in r["assign_link"]] == \
        [(B, a, b) for a, b in zip(counts[:-1], counts[1:])]
    off = np.concatenate([[0], np.cumsum(counts)])
    for b in range(B):
        (a, obj, y) = _milp(det, links, new, end, counts, b)
        got = _gpu_rows(r, b)
        assert _same(got, a), (counts, b)
        assert abs(_objective(det[b], [l[b:b + 1] for l in links], new[b], end[b], got) - obj) < 1e-9
        mt = r["match"][b].cpu()
        for f in range(len(counts) - 1):
            m = mt[off[f]:off[f + 1]]
            al = got[1][f][0]
            assert torch.equal(m >= 0, al.sum(1) > 0)
            assert torch.equal(m[m >= 0].long(), al.argmax(1)[m >= 0])
        if gap and b == 0:
            (_, obj2, _) = _milp(det, links, new, end, counts, b, exclude=y)
            assert obj - obj2 > 1e-7, (obj, obj2)


@pytest.mark.gpu
@pytest.mark.parametrize("n,m", [(1, 1), (3, 2), (8, 8), (7, 19), (64, 64), (128, 128)])
def test_flow_equals_lp_assign_at_two_frames(n, m):
    """K = 2: the min-cost flow and the assignment solver (mmmot_lp_assign), two exact solvers, agree bit for bit on
    unique-optimum instances."""
    import mmmot_b200
    g = torch.Generator().manual_seed(7 * n + m)
    B = 6
    det, links, new, end = _rand_frames(g, [n, m], B)
    det, links, new, end = det.cuda(), [links[0].cuda()], new.cuda(), end.cuda()
    rf = mmmot_b200.solve_frames(det, links, new, end, [n, m])
    rl = mmmot_b200.solve_batch(det, links[0], new, end, n, m)
    for k in ("assign_det", "assign_new", "assign_end", "match"):
        assert torch.equal(rf[k], rl[k]), k
    assert torch.equal(rf["assign_link"][0], rl["assign_link"])


@pytest.mark.gpu
def test_flow_large_feasible_and_optimal():
    """K = 5 with 128 detections per frame: the flow constraints of solvers.py:83-111 hold and the objective equals
    the MILP optimum."""
    import mmmot_b200
    counts = [128] * 5
    g = torch.Generator().manual_seed(5128)
    B = 2
    det, links, new, end = _rand_frames(g, counts, B)
    r = mmmot_b200.solve_frames(det.cuda(), [l.cuda() for l in links], new.cuda(), end.cuda(), counts)
    for b in range(B):
        got = _gpu_rows(r, b)
        assert _feasible(got, counts)
        (_, obj, _) = _milp(det, links, new, end, counts, b)
        assert abs(_objective(det[b], [l[b:b + 1] for l in links], new[b], end[b], got) - obj) < 1e-8


@pytest.mark.gpu
@pytest.mark.parametrize("counts", [(3, 5, 2), (4, 4, 4, 4), (1, 6, 6, 1, 3), (16, 16, 16), (12, 1, 9, 12, 5, 12, 3, 12)])
def test_flow_ties_deterministic_and_optimal(counts):
    """Integer-valued scores (ties everywhere, paths of profit exactly 0): the result is feasible, its objective is the
    MILP optimum, two runs are bit-identical, and it is the solution the documented tie rules pick (smaller node index
    first, no zero-profit augmentation), i.e. bit for bit the numpy restatement's."""
    import mmmot_b200
    counts = list(counts)
    g = torch.Generator().manual_seed(sum(counts) + len(counts))
    B = 4
    det, links, new, end = _rand_frames(g, counts, B, scale=2)
    args = (det.cuda(), [l.cuda() for l in links], new.cuda(), end.cuda(), counts)
    r1 = mmmot_b200.solve_frames(*args)
    r2 = mmmot_b200.solve_frames(*args)
    for k in ("assign_det", "assign_new", "assign_end", "match"):
        assert torch.equal(r1[k], r2[k]), k
    assert all(torch.equal(a, b) for a, b in zip(r1["assign_link"], r2["assign_link"]))
    for b in range(B):
        got = _gpu_rows(r1, b)
        assert _feasible(got, counts)
        (_, obj, _) = _milp(det, links, new, end, counts, b)
        assert abs(_objective(det[b], [l[b:b + 1] for l in links], new[b], end[b], got) - obj) < 1e-9
        assert _same(got, flow_rehearsal(det[b], [l[b] for l in links], new[b], end[b], counts)), b


def _cap_counts(L, K):
    """K frames alternating 1 and n detections, the last frame topped up to L in all: large L, few link variables."""
    counts = [1 if f % 2 == 0 else 0 for f in range(K)]
    n = (L - sum(counts)) // (K // 2)
    counts = [c or n for c in counts]
    counts[-1] += L - sum(counts)
    return counts


@pytest.mark.gpu
@pytest.mark.parametrize("L,K,B,warps", [(1202, 4, 4, 3), (2000, 6, 3, 2), (4469, 64, 2, 1)])
def test_flow_large_samples_up_to_the_shared_memory_cap(L, K, B, warps):
    """Samples whose state takes 1 to 3 warps' share of one SM's shared memory, up to the largest L the cap admits
    (4469 detections, a 232432-byte slab, one warp per CTA): bit-exact against the MILP.  Sparse profitable scores
    (about 2 % of the detections worth a track) keep the augmentation count, and so the run time, small."""
    import mmmot_b200
    counts = _cap_counts(L, K)
    assert sum(counts) == L and 232448 // ((52 * L + 42 + 15) // 16 * 16) == warps
    g = torch.Generator().manual_seed(L)
    det = torch.rand(B, L, generator=g) - 0.99
    new, end = torch.rand(B, L, generator=g) * 0.01, torch.rand(B, L, generator=g) * 0.01
    new[:, :counts[0]] = 0
    end[:, L - counts[-1]:] = 0
    links = [torch.rand(B, a, b, generator=g) * 0.02 for a, b in zip(counts[:-1], counts[1:])]
    r = mmmot_b200.solve_frames(det.cuda(), [l.cuda() for l in links], new.cuda(), end.cuda(), counts)
    for b in range(B):
        (a, obj, _) = _milp(det, links, new, end, counts, b)
        got = _gpu_rows(r, b)
        assert a[0].sum() > 0 and _same(got, a), b
        assert abs(_objective(det[b], [l[b:b + 1] for l in links], new[b], end[b], got) - obj) < 1e-8


@pytest.mark.gpu
def test_predict_three_frame_windows_end_to_end(tmp_path):
    """A synthetic 5-frame sequence in 3-frame windows (frames 0-2, 2-4) through TrackingModule.predict on the
    outputs of TrackingNet.forward: the stitched ids and the KITTI text equal those of the same host code fed the MILP's
    assignment of the same GPU scores."""
    import mmmot_b200
    from mmmot_b200.synthetic import synthetic_pair, synthetic_state_dict
    from mmmot_b200.tracking_model import write_kitti_result
    net = mmmot_b200.TrackingNet(3, appear_skippool=True, score_arch="branch_cls", score_fusion_arch="C",
                                 affinity_op="multiply", softmax_mode="none", neg_threshold=0.2, test_mode=2, dropblock=0)
    net.load_state_dict(synthetic_state_dict("C", seed=0))
    net.cuda().eval()

    class Recorder:
        """The network, keeping the scores of its last forward."""
        test_mode = net.test_mode

        def eval(self):
            net.eval()

        def __call__(self, *a):
            self.out = net(*a)
            return self.out
    rec = Recorder()
    tm = mmmot_b200.TrackingModule(rec, None, None, det_type="3D")
    tm.eval()
    ref = mmmot_b200.TrackingModule(rec, None, None, det_type="3D")
    ref.eval()
    counts = [6, 4, 7, 5, 6]
    frames = []
    for t, n in enumerate(counts):
        crops, det_info, _ = synthetic_pair(n // 2, n - n // 2, 16, 32, seed=10 + t)    # n detections of one frame
        g = torch.Generator().manual_seed(50 + t)
        frames.append((crops, det_info, {
            "name": torch.zeros(1, n).long(), "truncated": torch.zeros(1, n), "occluded": torch.zeros(1, n).long(),
            "alpha": torch.zeros(1, n), "bbox": torch.rand(1, n, 4, generator=g) * 100,
            "dimensions": torch.rand(1, n, 3, generator=g), "location": torch.rand(1, n, 3, generator=g) * 30,
            "rotation_y": torch.zeros(1, n), "frame_idx": torch.tensor([t])}))
    for w in (0, 2):
        win = frames[w:w + 3]
        crops = torch.cat([c for c, _, _ in win]).cuda()
        pts, sp, base = [], [torch.zeros(1)], 0.0
        for _, info, _ in win:
            pts.append(info["points"][0])
            sp.append(info["points_split"][0][1:] + base)
            base += float(info["points_split"][0][-1])
        info = {"points": torch.cat(pts)[None].cuda(), "points_split": torch.cat(sp)[None].cuda()}
        split = [torch.tensor([counts[w + i]]) for i in range(3)]
        ids, out, start = tm.predict(crops, info, [copy.deepcopy(d) for _, _, d in win], split)
        assert start == (0 if w == 0 else 1)
        det, link, new, end, _ = rec.out
        t = net.test_mode
        (a, _, _) = lp_ref.milp_solve(det[t].cpu(), [l[t:t + 1].cpu() for l in link], new[t].cpu(), end[t].cpu(),
                                      [int(s) for s in split])
        rids, rboxes = ref.assign_det_id(*a, split, [copy.deepcopy(d) for _, _, d in win])
        rout = ref.align_id(rids, rboxes)
        assert [[int(v) for v in x] for x in ids] == [[int(v) for v in x] for x in rout[0]]
    assert [[int(v) for v in x] for x in tm.frames_id] == [[int(v) for v in x] for x in ref.frames_id]
    assert sum(len(x) for x in tm.frames_id) > 0
    write_kitti_result(str(tmp_path / "gpu"), "0000", "step", tm.frames_id, copy.deepcopy(tm.frames_det), part="val")
    write_kitti_result(str(tmp_path / "milp"), "0000", "step", ref.frames_id, copy.deepcopy(ref.frames_det), part="val")
    text = (tmp_path / "gpu" / "step" / "val" / "0000.txt").read_text()
    assert text and text == (tmp_path / "milp" / "step" / "val" / "0000.txt").read_text()
