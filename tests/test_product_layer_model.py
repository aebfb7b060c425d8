"""CPU model of the layer boundaries of the batched product-circuit proofs (spartan_b200/csrc/snark.cpp batched_prove), against the oracle.

- Tail: the launch that folds the tables to two entries publishes them, and the host binds the last variable itself: claim = a0 + r (a1 - a0),
  which must be the value the reference reads after its last bound_poly_var_top (product_tree.rs:336-345).
- Head: the eq table of a layer without eq-factoring is built from E = eq(rand[1..], .) before r_layer is known, then extended by the top
  variable as [(1 - r_layer) E | r_layer E].
- Switch: after the eq-factored rounds 0 .. jG-1 the standard rounds run on C' = eq(rand[jG..], .), the last suffix table, instead of the
  reference's bound C = prefix * eq(rand[jG..], .); the host multiplies the product instances' evaluations by prefix (dot-product instances,
  which carry their own weight table, are not scaled), and the combined round polynomials must be the reference's."""
import random

from oracle.spartan_ref import core as oc

Q = oc.Q


def rand_arr(rnd, n):
    return oc.to_arr([rnd.randrange(Q) for _ in range(n)])


def eq_factor(tau, r):
    return ((1 - tau) + r * (2 * tau - 1)) % Q


def test_two_entry_claim_is_the_last_fold():
    rnd = random.Random(5)
    for n in (1, 2, 5):
        A = rand_arr(rnd, 1 << n)
        rs = [rnd.randrange(Q) for _ in range(n)]
        for r in rs[:-1]:
            A = oc.bound_top(A, r)
        a0, a1 = oc.to_ints(A)
        claim = (a0 + rs[-1] * (a1 - a0)) % Q
        assert claim == oc.arr_get(oc.bound_top(A.copy(), rs[-1]), 0)
    # the edges of the subtraction: a1 = a0, a1 < a0, and r = 0, 1, q - 1
    for a0, a1 in ((0, 0), (7, 7), (Q - 1, 0), (0, Q - 1), (123, 5)):
        for r in (0, 1, Q - 1, 2):
            assert (a0 + r * (a1 - a0)) % Q == oc.arr_get(oc.bound_top(oc.to_arr([a0, a1]), r), 0)


def test_eq_table_extended_by_the_top_variable():
    rnd = random.Random(6)
    for n in (0, 1, 4):
        tail = [rnd.randrange(Q) for _ in range(n)]
        for r in (rnd.randrange(Q), 0, 1):
            E = oc.to_ints(oc.eq_evals(tail))
            hi = [e * r % Q for e in E]
            lo = [(e - h) % Q for e, h in zip(E, hi)]
            assert lo + hi == oc.to_ints(oc.eq_evals([r] + tail))


def test_prefix_on_the_host_after_the_switch():
    rnd = random.Random(7)
    n, jG, n_prod, n_dotp = 7, 3, 3, 2
    tau = [rnd.randrange(Q) for _ in range(n)]
    A = [rand_arr(rnd, 1 << n) for _ in range(n_prod + n_dotp)]
    B = [rand_arr(rnd, 1 << n) for _ in range(n_prod + n_dotp)]
    W = [rand_arr(rnd, 1 << n) for _ in range(n_dotp)]          # the dot-product circuits' own weight tables
    coeff = [rnd.randrange(Q) for _ in range(n_prod + n_dotp)]
    C = oc.eq_evals(tau)                                         # the reference's shared C, bound every round
    prefix = 1
    for j in range(jG):                                          # the eq-factored rounds (their bookkeeping: test_eqfactor_model.py)
        r = rnd.randrange(Q)
        prefix = prefix * eq_factor(tau[j], r) % Q
        A = [oc.bound_top(a, r) for a in A]
        B = [oc.bound_top(b, r) for b in B]
        W = [oc.bound_top(w, r) for w in W]
        C = oc.bound_top(C, r)
    # C' = the last suffix table, E_{jG-1}: the sum over the top jG-1 index bits of E_0 = eq(tau[1..], .) (k_eq_suffix)
    E0 = oc.to_ints(oc.eq_evals(tau[1:]))
    sz = len(E0) >> (jG - 1)
    Cs = oc.to_arr([sum(E0[b * sz + y] for b in range(1 << (jG - 1))) % Q for y in range(sz)])
    assert oc.to_ints(Cs) == oc.to_ints(oc.eq_evals(tau[jG:]))
    assert [prefix * c % Q for c in oc.to_ints(Cs)] == oc.to_ints(C)
    coeff_std = [c * prefix % Q for c in coeff[:n_prod]] + coeff[n_prod:]
    for j in range(jG, n):
        ref = [oc.sc_eval_cubic(A[i], B[i], C) for i in range(n_prod)] + [oc.sc_eval_cubic(A[n_prod + i], B[n_prod + i], W[i]) for i in range(n_dotp)]
        dev = [oc.sc_eval_cubic(A[i], B[i], Cs) for i in range(n_prod)] + ref[n_prod:]
        for k in range(3):
            assert sum(ev[k] * c for ev, c in zip(dev, coeff_std)) % Q == sum(ev[k] * c for ev, c in zip(ref, coeff)) % Q
        r = rnd.randrange(Q)
        A = [oc.bound_top(a, r) for a in A]
        B = [oc.bound_top(b, r) for b in B]
        W = [oc.bound_top(w, r) for w in W]
        C = oc.bound_top(C, r)
        Cs = oc.bound_top(Cs, r)
