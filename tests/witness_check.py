"""TEST INFRASTRUCTURE ONLY -- an independent witness checker over Python ints, for the library's witness check
(csrc/check.cu, ``Prover.check_arrays``).  It shares no code with the library: sigma comes from a dict of the 3n cell
labels, the lookup from a set of table rows and the shuffle from two Counters.  ``check`` returns what the library
returns: five counts and, per category, the lowest ``limit`` locations in ascending order (copy: (c, sigma(c)) pairs)."""
from __future__ import annotations

from collections import Counter

R = 21888242871839275222246405745257275088548364400416034343698204186575808495617


def _roots(n):
    w = pow(5, (R - 1) // n, R)
    out, x = [], 1
    for _ in range(n):
        out.append(x)
        x = x * w % R
    return out


def _monomial(exps, vals):
    m = 1
    for x, e in zip(vals, exps):
        m = m * pow(x, e, R) % R
    return m


def check(n, Q, S, A, B, C, public, custom=(), lookup=None, shuffle=None, limit=16):
    """Q: {"QL", "QR", "QM", "QO", "QC"} -> n ints; S: (S1, S2, S3) n ints each; A, B, C: n ints (shorter ones are zero
    padded); custom: [(3 or 6 exponents, n ints)]; lookup: (q_K, Q_T or None, table rows as (t1, t2, t3[, t4]) tuples);
    shuffle: (q_in, q_out).  -> {"counts": [gate, copy, key, lookup, shuffle], "gate": rows, "copy": [(c, sigma(c))],
    "key": cells, "lookup": rows, "shuffle": rows}, lists cut at ``limit``"""
    W = [[int(v) % R for v in X] + [0] * (n - len(X)) for X in (A, B, C)]
    pi = [(-int(v)) % R for v in public] + [0] * (n - len(public))
    found = {k: [] for k in ("gate", "copy", "key", "lookup", "shuffle")}
    for i in range(n):
        a, b, c = (w[i] for w in W)
        nxt = tuple(w[(i + 1) % n] for w in W)
        g = (a * Q["QL"][i] + b * Q["QR"][i] + a * b * Q["QM"][i] + c * Q["QO"][i] + Q["QC"][i] + pi[i]) % R
        for exps, col in custom:
            g = (g + int(col[i]) * _monomial(exps, (a, b, c) + nxt)) % R
        if g:
            found["gate"].append(i)
    roots = _roots(n)
    label = {roots[r] * (k + 1) % R: 3 * r + k for r in range(n) for k in range(3)}
    named = set()
    for cell in range(3 * n):
        row, col = divmod(cell, 3)
        target = label.get(int(S[col][row]) % R)
        if target is None or target in named:
            found["key"].append(cell)
        if target is not None:
            named.add(target)
            trow, tcol = divmod(target, 3)
            if W[col][row] != W[tcol][trow]:
                found["copy"].append((cell, target))
    if lookup is not None:
        qk, qt, rows = lookup
        table = {tuple(int(x) % R for x in t) + ((0,) if len(t) == 3 else ()) for t in rows}
        for i in range(n):
            key = (W[0][i], W[1][i], W[2][i], int(qt[i]) if qt is not None else 0)
            if qk[i] and key not in table:
                found["lookup"].append(i)
    if shuffle is not None:
        q_in, q_out = shuffle
        tup = lambda i: (W[0][i], W[1][i], W[2][i])  # noqa: E731
        cin = Counter(tup(i) for i in range(n) if q_in[i])
        cout = Counter(tup(i) for i in range(n) if q_out[i])
        found["shuffle"] = [i for i in range(n) if (q_in[i] or q_out[i]) and cin[tup(i)] != cout[tup(i)]]
    out = {"counts": [len(found[k]) for k in ("gate", "copy", "key", "lookup", "shuffle")]}
    out.update((k, v[:limit]) for k, v in found.items())
    return out


def check_circuit(c, A, B, C, public, S=None, limit=16):
    """``check`` for a plonkathon_b200.synthetic.ArrayCircuit (S: its permutation columns unless given)"""
    from plonkathon_b200 import synthetic as syn
    from plonkathon_b200.lookup import check_lookups, padded_table
    n = c.group_order
    S = S or syn.permutation_polys(c.wire_L, c.wire_R, c.wire_O, n, c.n_constraints)
    Q = {"QL": c.QL, "QR": c.QR, "QM": c.QM, "QO": c.QO, "QC": c.QC}
    lookup = None
    if c.lookup or c.lookups:
        qk, qtag, cols, rows = check_lookups(c.lookups or [c.lookup], n)
        lookup = (qk, qtag if c.lookups else None, list(zip(*[col[:rows] for col in cols])))
    return check(n, Q, S, A, B, C, public, c.custom, lookup, c.shuffle or None, limit)


def copy_failures(wire_L, wire_R, wire_O, n, n_constraints, changed):
    """The copy category of a valid witness after the cells ``changed`` (a bool array over the 3n cells) were given new
    values, for circuits too large for ``check``: every changed cell of one variable must hold the same new value (so a
    cell fails iff exactly one of it and sigma(it) changed).  sigma from the wire ids with numpy, as
    ``synthetic.permutation_polys`` groups them.  -> sorted (c, sigma(c)) pairs, as an (k, 2) int64 array"""
    import numpy as np
    ids = np.full((n, 3), -1, dtype=np.int64)
    for col, w in enumerate((wire_L, wire_R, wire_O)):
        ids[:n_constraints, col] = np.asarray(w)[:n_constraints]
    flat = ids.reshape(-1)
    order = np.argsort(flat, kind="stable")
    start = np.ones(len(order), dtype=bool)
    start[1:] = flat[order][1:] != flat[order][:-1]
    prev = np.empty(len(order), dtype=np.int64)
    prev[1:] = order[:-1]
    first = np.flatnonzero(start)
    last = np.append(first[1:], len(order)) - 1
    prev[first] = order[last]
    sigma = np.empty(len(order), dtype=np.int64)
    sigma[order] = prev
    cells = np.flatnonzero(changed != changed[sigma])
    return np.stack([cells, sigma[cells]], axis=1)
