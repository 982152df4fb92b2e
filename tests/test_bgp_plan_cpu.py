"""CPU: the plan of kb_bgp_execute's component route (kolibrie_b200/csrc/kb_bgp_plan.hpp), built on the host with g++ from the same
header the library compiles. tests/cpp/bgp_plan_driver.cpp plans thousands of random BGP hypergraphs — paths, trees, stars with arms,
cycles, disconnected unions, patterns without variables, and random mixtures — and this test checks that the components are the
connected components, that GYO's verdict equals a brute-force search for a join tree (every labelled tree, running intersection),
that no join inside a component is keyless, and that an acyclic component's order walks its join tree from its smallest relation."""
import itertools
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "kolibrie_b200", "csrc")


def build_driver(out_dir):
    """builds tests/cpp/bgp_plan_driver.cpp into out_dir (the repository tree may be read-only)"""
    exe = os.path.join(str(out_dir), "bgp_plan_driver")
    cmd = ["/usr/bin/g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-I", CSRC, "-o", exe, os.path.join(ROOT, "tests", "cpp", "bgp_plan_driver.cpp")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    return exe


def shape(rng, kind, base):
    """variables (at most 3 per pattern, as a triple pattern has) of one connected shape, with variable ids from `base`"""
    if kind == "path":
        n = int(rng.integers(2, 9))
        return [[base + i, base + i + 1] for i in range(n)]
    if kind == "tree":
        n = int(rng.integers(2, 10))
        return [[base + int(rng.integers(0, i + 1)), base + i + 1] for i in range(n)]
    if kind == "star":  # a hub variable with arms of length 1..3
        pats, nxt = [], base + 1
        for _ in range(int(rng.integers(2, 5))):
            prev = base
            for _ in range(int(rng.integers(1, 4))):
                pats.append([prev, nxt])
                prev, nxt = nxt, nxt + 1
        return pats
    if kind == "cycle":
        n = int(rng.integers(3, 7))
        return [[base + i, base + (i + 1) % n] for i in range(n)]
    if kind == "const":
        return [[]]
    # random: 1-3 variables per pattern over a small pool (cycles, repeated sets, triangles covered by a wider pattern)
    n, pool = int(rng.integers(1, 7)), int(rng.integers(1, 6))
    return [sorted(set(int(x) + base for x in rng.integers(0, pool, int(rng.integers(1, 4))))) for _ in range(n)]


def random_bgp(rng):
    pats, base = [], 0
    for _ in range(int(rng.integers(1, 4))):
        kind = str(rng.choice(["path", "tree", "star", "cycle", "const", "random", "random"]))
        part = shape(rng, kind, base)
        if len(pats) + len(part) > 16:
            break
        pats += part
        base += 20
    perm = rng.permutation(len(pats))  # textual order is not the join order
    pats = [pats[i] for i in perm]
    rows = [int(x) for x in rng.integers(1, 50, len(pats))]
    return pats, rows


def components(pats):
    n, comp = len(pats), [-1] * len(pats)
    out = []
    for s in range(n):
        if comp[s] >= 0:
            continue
        comp[s], todo, members = len(out), [s], []
        while todo:
            k = todo.pop()
            members.append(k)
            for j in range(n):
                if comp[j] < 0 and set(pats[k]) & set(pats[j]):
                    comp[j] = len(out)
                    todo.append(j)
        out.append(sorted(members))
    return out


def prufer_trees(m):
    """every labelled tree on m nodes, as edge lists"""
    if m == 1:
        yield []
        return
    for seq in itertools.product(range(m), repeat=m - 2):
        degree = [1] * m
        for x in seq:
            degree[x] += 1
        edges = []
        for x in seq:
            leaf = min(i for i in range(m) if degree[i] == 1)
            edges.append((leaf, x))
            degree[leaf] -= 1
            degree[x] -= 1
        u, v = [i for i in range(m) if degree[i] == 1]
        edges.append((u, v))
        yield edges


def running_intersection(sets, edges):
    """every variable's patterns induce a connected subtree of the tree `edges`"""
    for v in set().union(*sets):
        nodes = {i for i, s in enumerate(sets) if v in s}
        start = next(iter(nodes))
        seen, todo = {start}, [start]
        while todo:
            a = todo.pop()
            for x, y in edges:
                for p, q in ((x, y), (y, x)):
                    if p == a and q in nodes and q not in seen:
                        seen.add(q)
                        todo.append(q)
        if seen != nodes:
            return False
    return True


def brute_acyclic(sets):
    return any(running_intersection(sets, t) for t in prufer_trees(len(sets)))


def test_plan_against_brute_force(tmp_path):
    exe = build_driver(tmp_path)
    rng = np.random.default_rng(7)
    cases = [random_bgp(rng) for _ in range(3000)]
    text = "\n".join(" ".join([str(len(p))] + [" ".join(str(x) for x in [len(q)] + q) for q in p] + [str(r) for r in rows]) for p, rows in cases)
    r = subprocess.run([exe], input=text + "\n", stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:]
    lines = r.stdout.split("\n")
    brute = {"acyclic": 0, "cyclic": 0}
    for (pats, rows), line in zip(cases, lines):
        tok = [int(x) for x in line.split()]
        n_comp, at = tok[0], 1
        want = components(pats)
        assert n_comp == len(want), (pats, line)
        for c in range(n_comp):
            size = tok[at]
            members = tok[at + 1: at + 1 + size]
            acyclic = tok[at + 1 + size] == 1
            at += 2 + size
            parent = {}
            if acyclic:
                parent = dict(zip(members, tok[at: at + size]))
                at += size
            n_order = tok[at]
            order = tok[at + 1: at + 1 + n_order]
            at += 1 + n_order
            assert members == want[c], (pats, line)
            sets = [set(pats[k]) for k in members]
            if size <= 6:
                truth = brute_acyclic(sets)
                assert acyclic == truth, (pats, members, acyclic)
                brute["acyclic" if truth else "cyclic"] += 1
            assert sorted(order) == members, (pats, order)
            assert order[0] == min(members, key=lambda k: (rows[k], k)), "the order starts at the smallest relation"
            for i in range(1, len(order)):
                held = set().union(*(set(pats[k]) for k in order[:i]))
                assert held & set(pats[order[i]]), f"keyless join inside a component: {pats} order {order}"
            if acyclic:
                edges = [(k, p) for k, p in parent.items() if p >= 0]
                assert len(edges) == size - 1 and sum(p < 0 for p in parent.values()) == 1
                assert running_intersection([set(pats[k]) for k in members], [(members.index(a), members.index(b)) for a, b in edges]), (pats, parent)
                for i in range(1, len(order)):  # each step adds a tree neighbour of the patterns joined so far
                    assert any(parent[order[i]] == k or parent[k] == order[i] for k in order[:i]), (pats, order, parent)
        assert at == len(tok), line
    assert brute["acyclic"] > 500 and brute["cyclic"] > 100, brute
