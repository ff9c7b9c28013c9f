"""CPU restatement of how the damped-solve kernels choose their shared-memory storage (no GPU, no library).

Each solver keeps its matrix in shared memory and picks, by size, square fp64 (FULL), packed fp64 or packed fp32 storage, or rejects the
size with BANET_ERR_UNSUPPORTED (-4).  The rules below restate lm_step_smem / lm_step (lm_step.cu), arrow_smem / arrow_plan
(lm_window_batch.cu), lm_solve_uses_double / lm_solve_update (lm_solve.cu) and solve_bwd_floats / launch_solve_bwd (lm_bwd.cu).
tests/test_solve_edges.py ties the rejection edges to the built library and runs every variant on the GPU at the sizes generated here.

C is the lambda-MLP width; the MLP buffers share the solver's shared memory, so C moves the switches.  Where lambda is given:
  * banet_lm_step and the dense window pass C = 1 (lm_step_smem still reserves max(4C, 1024) floats of slice partials);
  * the arrow (banet_lm_window_batch_solve_update and its backward) reserves nothing: Cm = 0.
"""
STEP_NB = 4
KB = 1024
SQUARE64, PACKED64, PACKED32, REJECT = "square_fp64", "packed_fp64", "packed_fp32", "rejected"


def _mlp_bytes(C):
    return (8 * C + max(4 * C, 1024)) * 4


def lm_step_smem(P, C, dbl, full):
    nA = ((P + 1) * ((P + 1) | 1) if full else (P + 1) * (P + 2) // 2) + 2 * P + STEP_NB
    return nA * (8 if dbl else 4) + _mlp_bytes(C)


def lm_step_plan(P, C):
    """lm_step_kernel<S, FULL> for P = 6 + K unknowns (or the dense window's 6 nf + K) at MLP width C (1 when lambda is given)."""
    if lm_step_smem(P, C, True, True) <= 200 * KB:
        return SQUARE64
    if lm_step_smem(P, C, True, False) <= 200 * KB:
        return PACKED64
    return PACKED32 if lm_step_smem(P, C, False, False) <= 220 * KB else REJECT


def arrow_smem(K, C, dbl, full):
    nA = (K + 1) * ((K + 1) | 1) if full else (K + 1) * (K + 2) // 2
    return (nA + 9 * K + STEP_NB) * (8 if dbl else 4) + (_mlp_bytes(C) if C > 0 else 0)


def arrow_plan(K, C):
    """window_arrow_step_kernel / window_arrow_step_bwd_kernel <S, FULL> at depth size K; C = 0 when lambda is given (and in the backward)."""
    if K < 1 or K > 256:
        return REJECT
    if arrow_smem(K, C, True, True) <= 200 * KB:
        return SQUARE64
    if arrow_smem(K, C, True, False) <= 200 * KB:
        return PACKED64
    return PACKED32 if arrow_smem(K, C, False, False) <= 220 * KB else REJECT


def lm_solve_plan(P):
    """lm_solve_kernel<S> (banet_lm_solve_update, the pair training forward): packed only."""
    n = P * (P + 1) // 2 + 2 * P
    if n * 8 <= 200 * KB:
        return PACKED64
    return PACKED32 if n * 4 <= 220 * KB else REJECT


def solve_bwd_plan(P, forward_plan):
    """lm_solve_bwd_kernel<S>: factors in the precision its forward used (forward_plan = that forward's plan at the same P)."""
    n = P * (P + 1) // 2 + 3 * P
    if n * 4 > 220 * KB or forward_plan == REJECT:
        return REJECT
    return PACKED64 if forward_plan in (SQUARE64, PACKED64) else PACKED32


def pair_bwd_plan(P):
    """banet_lm_solve_update_bwd: the backward of lm_solve_update."""
    return solve_bwd_plan(P, lm_solve_plan(P))


def dense_window_bwd_plan(Pj):
    """banet_lm_window_solve_update_bwd: the backward of lm_step with lambda given on the assembled window (C = 1)."""
    return solve_bwd_plan(Pj, lm_step_plan(Pj, 1))


def switches(plan, lo, hi):
    """[(last size of one variant, first size of the next, (variant, next variant))] over lo..hi."""
    out, prev = [], plan(lo)
    for n in range(lo + 1, hi + 1):
        cur = plan(n)
        if cur != prev:
            out.append((n - 1, n, (prev, cur)))
            prev = cur
    return out


# every kernel and every C that moves its switches: name -> (plan of the size, the range searched)
PLANS = {
    "lm_step_lambda_given": (lambda P: lm_step_plan(P, 1), (7, 400)),
    "lm_step_mlp_C5": (lambda P: lm_step_plan(P, 5), (7, 400)),
    "lm_step_mlp_C128": (lambda P: lm_step_plan(P, 128), (7, 400)),
    "lm_step_mlp_C256": (lambda P: lm_step_plan(P, 256), (7, 400)),
    "arrow_lambda_given": (lambda K: arrow_plan(K, 0), (1, 300)),
    "arrow_mlp_C5": (lambda K: arrow_plan(K, 5), (1, 300)),
    "arrow_mlp_C128": (lambda K: arrow_plan(K, 128), (1, 300)),
    "arrow_mlp_C256": (lambda K: arrow_plan(K, 256), (1, 300)),
    "lm_solve": (lm_solve_plan, (7, 400)),
    "lm_solve_bwd_pairs": (pair_bwd_plan, (7, 400)),
    "lm_solve_bwd_dense_window": (dense_window_bwd_plan, (7, 400)),
}


def edge_sizes(name):
    """The sizes on both sides of every switch of one plan, with each residue mod 4 present among the accepted sizes."""
    plan, (lo, hi) = PLANS[name]
    sizes = set()
    for a, b, _ in switches(plan, lo, hi):
        sizes.update((a, b))
    accepted = sorted(s for s in sizes if plan(s) != REJECT)
    for r in range(4):
        if not any(s % 4 == r for s in accepted):
            s = max(accepted)
            while s % 4 != r or plan(s) == REJECT:
                s -= 1
            sizes.add(s)
    return sorted(sizes)


def rejection_edge(name):
    """(largest accepted size, smallest rejected size) of a plan."""
    plan, (lo, hi) = PLANS[name]
    rej = [b for a, b, (_, nxt) in switches(plan, lo, hi) if nxt == REJECT]
    assert len(rej) == 1, (name, rej)
    return rej[0] - 1, rej[0]
