"""CPU restatement of how the damped-solve kernels choose their shared-memory storage (no GPU, no library).

There are two solvers, each keeping its matrix in shared memory: lm_step_kernel (lm_step.cu; with its backward it is also banet_lm_solve_update,
its backward, and the dense keyframe window in both directions) and the arrow's window_arrow_step(_bwd)_kernel (lm_window_batch.cu).  Each
picks, by size, square fp64 (FULL), packed fp64 or packed fp32 storage, or rejects the size with BANET_ERR_UNSUPPORTED (-4).  The rules
below restate step_plan (lm_step.cu), arrow_plan (lm_window_batch.cu) and lm_lambda.  tests/test_solve_edges.py ties the rejection edges
to the built library and runs every variant on the GPU at the sizes generated here.

The storage variant depends on the matrix and its vectors alone.  The lambda-MLP's buffers share the matrix's storage (lm_step.cuh), so the
MLP width C (0 when lambda is given) enters only the rejection: shared memory is vectors + max(matrix, MLP buffers).
"""
STEP_NB = 4
KB = 1024
SQUARE64, PACKED64, PACKED32, REJECT = "square_fp64", "packed_fp64", "packed_fp32", "rejected"
MLP_ONLY = "mlp_only"


def mlp_bytes(C):
    return (8 * C + max(4 * C, 1024)) * 4 if C > 0 else 0


def _matrix(n, full):
    return (n + 1) * ((n + 1) | 1) if full else (n + 1) * (n + 2) // 2


def _plan(n, vectors, C):
    """The variant of a matrix of n unknowns with `vectors` elements of its type beside it, or REJECT."""
    if (_matrix(n, True) + vectors) * 8 <= 200 * KB:
        full, elem, variant = True, 8, SQUARE64
    elif (_matrix(n, False) + vectors) * 8 <= 200 * KB:
        full, elem, variant = False, 8, PACKED64
    else:
        full, elem, variant = False, 4, PACKED32
    return variant if max(_matrix(n, full) * elem, mlp_bytes(C)) + vectors * elem <= 220 * KB else REJECT


def step_plan(P, C=0):
    """lm_step_kernel / lm_step_bwd_kernel <S, FULL> for P = 6 + K unknowns (or the dense window's 6 nf + K); C: the MLP width, 0 when
    lambda is given."""
    return _plan(P, 2 * P + STEP_NB, C)


def arrow_plan(K, C=0):
    """window_arrow_step_kernel / window_arrow_step_bwd_kernel <S, FULL> at depth size K; C: the MLP width, 0 when lambda is given."""
    if K < 1 or K > 256:
        return REJECT
    return _plan(K, 9 * K + STEP_NB, C)


def lambda_plan(C):
    """banet_lm_lambda: the MLP's buffers alone."""
    return MLP_ONLY if mlp_bytes(C) <= 220 * KB else REJECT


def switches(plan, lo, hi):
    """[(last size of one variant, first size of the next, (variant, next variant))] over lo..hi."""
    out, prev = [], plan(lo)
    for n in range(lo + 1, hi + 1):
        cur = plan(n)
        if cur != prev:
            out.append((n - 1, n, (prev, cur)))
            prev = cur
    return out


# every C-ABI entry with a size edge: name -> (plan of the size, the range searched).  The size is P = 6 + K (the dense window's 6 nf + K),
# the arrow's K, or, for the *_width entries, the MLP width C.
PLANS = {
    "lm_step_lambda_given": (lambda P: step_plan(P), (7, 400)),
    "lm_step_mlp_C5": (lambda P: step_plan(P, 5), (7, 400)),
    "lm_step_mlp_C128": (lambda P: step_plan(P, 128), (7, 400)),
    "lm_step_mlp_C256": (lambda P: step_plan(P, 256), (7, 400)),
    "lm_step_width_P7": (lambda C: step_plan(7, C), (1, 6000)),
    "lm_step_width_P262": (lambda C: step_plan(262, C), (1, 6000)),
    "lm_lambda_width": (lambda_plan, (1, 6000)),
    "lm_solve": (lambda P: step_plan(P), (7, 400)),
    "lm_solve_bwd_pairs": (lambda P: step_plan(P), (7, 400)),
    "dense_window": (lambda P: step_plan(P), (7, 400)),
    "lm_solve_bwd_dense_window": (lambda P: step_plan(P), (7, 400)),
    "arrow_lambda_given": (lambda K: arrow_plan(K), (1, 300)),
    "arrow_bwd": (lambda K: arrow_plan(K), (1, 300)),
    "arrow_mlp_C5": (lambda K: arrow_plan(K, 5), (1, 300)),
    "arrow_mlp_C128": (lambda K: arrow_plan(K, 128), (1, 300)),
    "arrow_mlp_C256": (lambda K: arrow_plan(K, 256), (1, 300)),
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
