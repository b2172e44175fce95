"""CPU: the case table of the element-wise one-launch eval block test (tests/block_eval_cases.py)
reaches every compiled (tile geometry, expansion) pair of csrc/block_eval.cuh with both activation
classes, in the unsplit and the cluster launch (test_block_eval_fp64_gpu.py runs every case in the
plain, gate and pool modes of both), and every geometry over a multi-tile walk.  The pair list is
parsed out of the header, so a launch_eval<...> the tile plan never picks, or one without a case,
fails here; YAMB_BLOCK_EVAL_SOURCE points the parser at another copy of the header."""
import os

import pytest

import block_eval_cases as bc

SOURCE = os.environ.get("YAMB_BLOCK_EVAL_SOURCE") or bc.BLOCK_EVAL_SOURCE


def _grid():
    """Every shape the launcher accepts over a grid of sizes, with its plan."""
    for k in (3, 5, 7):
        for s in (1, 2):
            for expand in ((True, False) if k == 3 else (True,)):
                for cout in (8, 160, 168, 320):
                    for n in (1, 2, 3, 5):
                        for h in range(1, 40):
                            for w in range(1, 40, 3):
                                yield (n, h, w, cout, k, s, expand), bc.plan(n, h, w, cout, k, s, expand)


def test_instantiations_parse():
    inst = bc.compiled_instantiations(SOURCE)
    print("\n".join("%s %s" % (g, "expand" if ex else "no expansion") for g, ex in inst))
    assert len(inst) == 14, inst
    assert all(g.k in (3, 5, 7) and g.s in (1, 2) for g, _ in inst)


def test_every_compiled_pair_is_reachable():
    reached = {(g, ex) for _, (g, ex, _) in _grid()}
    unreachable = sorted(set(bc.compiled_instantiations(SOURCE)) - reached)
    assert unreachable == [], "compiled pairs the tile plan never picks: %s" % unreachable
    assert reached <= set(bc.compiled_instantiations(bc.BLOCK_EVAL_SOURCE))


def test_plan_agrees_with_engine():
    from yet_another_mobilenet_series_b200 import engine
    for (n, h, w, cout, k, s, expand), (_, _, nt) in _grid():
        assert nt == engine.eval_tiles(k, s, n, bc.out_size(h, s), bc.out_size(w, s), cout), \
            (n, h, w, cout, k, s)
    for c in bc.CASES:
        assert bc.case_plan(c)[2] == engine.eval_tiles(c.k, c.s, c.N, bc.out_size(c.H, c.s),
                                                       bc.out_size(c.W, c.s), c.Cout), c.name


def test_table_reaches_every_pair_class_and_split():
    have = {}
    for c in bc.CASES:
        g, ex, nt = bc.case_plan(c)
        have.setdefault((g, ex, bc.lean(c)), []).append(c.name)
    lines, missing = [], []
    for g, ex in bc.compiled_instantiations(SOURCE):
        for lean in (True, False):
            names = have.get((g, ex, lean), [])
            lines.append("%s %-12s %-7s %s" % (tuple(g), "expand" if ex else "no expansion",
                                               "lean" if lean else "generic", ", ".join(names)))
            if not names:
                missing.append((g, ex, lean))
    print("\n".join(lines))
    assert missing == [], "(geometry, expand, lean) without a case: %s" % missing


def test_every_pair_walks():
    walks = {}
    for c in bc.CASES:
        g, ex, nt = bc.case_plan(c)
        walks[(g, ex)] = max(walks.get((g, ex), 0), nt)
    short = [(g, ex, walks.get((g, ex), 0)) for g, ex in bc.compiled_instantiations(SOURCE)
             if walks.get((g, ex), 0) < bc.WALK_TILES]
    assert short == [], "pairs without a case of >= %d tiles: %s" % (bc.WALK_TILES, short)


def test_table_reaches_the_edges():
    cs = bc.CASES
    need = {
        "H and W cut by the tile": lambda c, g: bc.out_size(c.H, c.s) % g.toh and
        bc.out_size(c.W, c.s) % g.tow,
        "odd N on two images per tile": lambda c, g: g.ti == 2 and c.N % 2 == 1,
        "stride 2, odd H and W": lambda c, g: c.s == 2 and c.H % 2 and c.W % 2 and c.H > 1,
        "a single output pixel": lambda c, g: bc.out_size(c.H, c.s) * bc.out_size(c.W, c.s) == 1,
        "Cin 8": lambda c, g: c.Cin == 8,
        "Cin 24 (K padding)": lambda c, g: c.Cin == 24,
        "Cin 256 (four K panels)": lambda c, g: c.Cin == 256 and c.expand,
        "Cin 256 without expansion": lambda c, g: c.Cin == 256 and not c.expand,
        "Chid 8": lambda c, g: c.Chid == 8,
        "Chid 144 (partial last slice)": lambda c, g: c.Chid == 144,
        "Chid >= 1152": lambda c, g: c.Chid >= 1152,
        "Cout 8": lambda c, g: c.Cout == 8,
        "Cout 168 (first wide width)": lambda c, g: c.Cout == 168,
        "Cout 320 (two W3 halves)": lambda c, g: c.Cout == 320,
        "gamma / beta NULL": lambda c, g: not c.affine,
        "residual": lambda c, g: c.residual,
        "no residual": lambda c, g: not c.residual,
        "cluster larger than the slices": lambda c, g: c.cs > bc.slices(c),
        "cluster larger than the slices, no expansion": lambda c, g: c.cs > bc.slices(c) and
        not c.expand,
    }
    for a in range(5):
        need["act %d" % a] = lambda c, g, a=a: c.act == a
    for s in bc.CLUSTER_SIZES:
        need["cluster %d" % s] = lambda c, g, s=s: c.cs == s
        need["cluster %d over a walk" % s] = lambda c, g, s=s: c.cs == s and \
            bc.case_plan(c)[2] >= bc.WALK_TILES
    missing = [k for k, pred in need.items() if not any(pred(c, bc.case_plan(c)[0]) for c in cs)]
    assert missing == [], "edges no case reaches: %s" % missing


def test_cases_are_legal():
    for c in bc.CASES:
        assert c.Cin % 8 == 0 and c.Chid % 8 == 0 and c.Cout % 8 == 0, c.name
        assert c.Cin <= 256 and c.Cout <= 320, c.name
        assert c.expand or (c.Chid == c.Cin and c.k == 3), c.name
        assert not c.residual or (c.s == 1 and c.Cin == c.Cout), c.name
        assert c.cs in bc.CLUSTER_SIZES, c.name
    assert len({c.name for c in bc.CASES}) == len(bc.CASES)


def test_parser_sees_a_pair_the_plan_never_picks(tmp_path):
    """A launch_eval<...> added to the header that the tile plan cannot reach is reported."""
    with open(bc.BLOCK_EVAL_SOURCE) as f:
        src = f.read()
    extra = src.replace("namespace yamb {", "namespace yamb {\n// launch_eval<EvGeom<3, 1, 7, 14, 1, 4>, "
                        "true, CLUSTER>(p, a, st);", 1)
    p = tmp_path / "block_eval.cuh"
    p.write_text(extra)
    inst = bc.compiled_instantiations(str(p))
    assert (bc.Geom(3, 1, 7, 14, 1, 4), True) in inst
    reached = {(g, ex) for _, (g, ex, _) in _grid()}
    assert sorted(set(inst) - reached) == [(bc.Geom(3, 1, 7, 14, 1, 4), True)]

