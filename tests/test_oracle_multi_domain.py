"""The restated multi-plan layout of multi_domain_scenes.py against the oracle, and each mixed-geometry scene's facts.

The level sizes, quotas and cell grids the restatement computes equal the oracle's for every geometry the GPU file runs;
each scene reaches what it is built for: tile-less groups at every position, eight distinct geometries accepted up to the
8 x 32 level table, partial last FAST tiles, a later group driving the candidate slots, refusal pairs that split on the
level-select footprint alone, and capacity sequences that rebuild exactly where the rule says (11 tests, about 2 s)."""
import pytest

import oracle as O
import multi_domain_scenes as S

EIGHT_SETS = [(S.EIGHT_NF, sf, nl, S.FAST) for nl, sf in S.EIGHT_SETTINGS.values()]


def _geometries():
    """(params, W, H) of every group the GPU file runs"""
    out = [(S.TILELESS_PARAMS, W, H) for W, H in [S.TILELESS] + S.TILELESS_PARTNERS]
    out += [(p, W, H) for p in EIGHT_SETS for W, H in S.EIGHT]
    out += [(p, W, H) for p, spec in S.SMEM_SETS.values() for W, H, _ in spec]
    out += [(p, W, H) for p, (W, H) in S.SMEM_SMALLER.values()]
    for score, nf, a, b in S.REFUSAL_PAIRS.values():
        out += [((nf - 1, 1.2, 1, score), W, H) for W, H in (a, b)]
    out += [((1000, 1.2, 8, S.FAST), W, H) for W, H in S.CAP_GEOMS]
    out += [(S.LIMIT_PARAMS, W, H) for W, H, _ in S.LIMIT_GROUPS]
    out += [(p, W, H) for p in S.DOMAIN_PARAMS for W, H in S.PARTNERS]
    return out


def test_restated_levels_equal_the_oracle():
    seen = set()
    for params, W, H in _geometries():
        nf, sf, nl = params[:3]
        if (nf, sf, nl, W, H) in seen:
            continue
        seen.add((nf, sf, nl, W, H))
        p = O.make_params(nf, sf, nl, 1, 20)
        _, _, quota = S.levels(nf, sf, nl)
        assert quota == [p.quota[l] for l in range(nl)], (nf, sf, nl)
        lay = S.Layout(nf, sf, nl, W, H)
        assert lay.ok, (params, W, H, lay.refused)
        for l, L in enumerate(lay.levels):
            assert (L.w, L.h) == O.level_size(p, l, W, H), (params, W, H, l)
            rc, g = O.cell_grid(p, l, W, H, L.w, L.h)
            assert rc == 0
            assert (L.cols, L.rows, L.ncells) == (g.cols, g.rows, g.n_cells), (params, W, H, l)
            if L.ncells:
                assert (L.cw, L.ch) == (g.cell_w, g.cell_h), (params, W, H, l)


def test_tileless_group_has_no_tiles_and_no_cells():
    lay = S.Layout(*S.TILELESS_PARAMS[:3], *S.TILELESS)
    assert lay.ok and all(L.nftiles == 0 and L.ncells == 0 for L in lay.levels)
    assert S.empty_levels(S.TILELESS_PARAMS, *S.TILELESS) == list(range(S.TILELESS_PARAMS[2]))
    for W, H in S.TILELESS_PARTNERS:
        assert S.Layout(*S.TILELESS_PARAMS[:3], W, H).nftiles > 0
    where = set()
    for name, spec in S.TILELESS_CALLS.items():
        P = S.Plan(S.TILELESS_PARAMS, spec)
        assert P.refused is None
        idx = [i for i, (W, H, _) in enumerate(spec) if (W, H) == S.TILELESS]
        for k, g in enumerate(P.groups):
            if (g["W"], g["H"]) == S.TILELESS:
                # a zero-length work range shares its start with the group after it (or ends the call's work)
                nxt = P.groups[k + 1] if k + 1 < len(P.groups) else dict(fwork0=P.nfwork, cwork0=P.ncwork)
                assert g["fwork0"] == nxt["fwork0"] and g["cwork0"] == nxt["cwork0"]
        if idx == [0]:
            where.add("first")
        elif idx == [len(spec) - 1]:
            where.add("last")
        elif len(idx) == 2 and idx[1] == idx[0] + 1:
            where.add("twice")
        else:
            where.add("middle")
    assert where == {"first", "middle", "last", "twice"}


def test_tileless_frame_on_the_oracle():
    nf, sf, nl, score, th = S.TILELESS_PARAMS
    from orb_slam_b200.synth import textured_frame
    rc, k, d, _ = O.extract(O.make_params(nf, sf, nl, score, th), textured_frame(*S.TILELESS, seed=3))
    assert rc == 0 and len(k) == 0 and len(d) == 0


def test_eight_groups_fill_the_level_table():
    assert len(set(S.EIGHT)) == S.MAX_GROUPS == len(S.EIGHT_BATCH)
    assert max(nl for nl, _ in S.EIGHT_SETTINGS.values()) == S.MAX_LEVELS
    for p in EIGHT_SETS:
        P = S.Plan(p, S.spec_of(S.EIGHT, S.EIGHT_BATCH))
        assert P.refused is None and len(P.groups) == S.MAX_GROUPS, p
    assert sum(S.Layout(S.EIGHT_NF, 1.2, 8, W, H).partial_tiles() for W, H in S.EIGHT) >= 4
    assert S.Layout(S.EIGHT_NF, 1.2, 8, 1241, 376).partial_tiles()


def test_a_later_group_drives_the_candidate_slots():
    drivers = {name: S.Plan(S.TILELESS_PARAMS, spec).cand_total[1] for name, spec in S.TILELESS_CALLS.items()}
    assert drivers["first"] == 2 and drivers["twice"] == 3
    assert S.Plan((S.EIGHT_NF, 3.0, 2, S.FAST), S.spec_of(S.EIGHT, S.EIGHT_BATCH)).smem()[1] == 5


@pytest.mark.parametrize("key", sorted(S.SMEM_SETS))
def test_level_select_sets_pass_48k(key):
    params, spec = S.SMEM_SETS[key]
    P = S.Plan(params, spec)
    assert P.refused is None and P.smem()[0] > S.SMEM_DEFAULT
    p2, (W, H) = S.SMEM_SMALLER[key]
    assert p2[3] == params[3]
    small = S.Plan(p2, [(W, H, 1)]).smem()[0]
    assert S.SMEM_DEFAULT < small < P.smem()[0]


@pytest.mark.parametrize("key", sorted(S.REFUSAL_PAIRS))
def test_refusal_pairs_split_exactly(key):
    """At nf the first geometry runs and the second is refused for its level-select footprint alone; one fewer runs both;
    in both orders the refusal names the second geometry's group."""
    score, nf, a, b = S.REFUSAL_PAIRS[key]
    assert S.first_refused(*b, 1.2, 1, score, lo=nf - 200) == nf
    assert S.first_refused(*a, 1.2, 1, score, lo=nf - 200) > nf
    for n in (nf - 1, nf):
        for W, H in (a, b):
            assert S.Layout(n, 1.2, 1, W, H).ok
    for order, named in (((a, b), 1), ((b, a), 0)):
        spec = [(W, H, 1) for W, H in order]
        assert S.Plan((nf - 1, 1.2, 1, score), spec).refused is None
        assert S.Plan((nf, 1.2, 1, score), spec).refused == (named, "level-select")
        # the largest kept list over the groups, checked once, would refuse without naming a group
        assert S.Plan((nf, 1.2, 1, score), spec[1 - named:2 - named]).refused is None


def test_capacity_sequences_rebuild_where_the_rule_says():
    calls = [S.spec_of(S.CAP_GEOMS, b) for b in S.CAP_SEQUENCE]
    res = S.capacity(calls)
    builds = 0
    for (rebuilt, cap), b in zip(res, S.CAP_SEQUENCE):
        builds += rebuilt
        assert all(x >= y for x, y in zip(cap, b))
    assert [sum(r for r, _ in res[:i + 1]) for i in range(len(res))] == S.CAP_BUILDS
    assert res[-1][1] == list(S.CAP_MAX)
    # without the growth rule (capacities = the call's frames) the sequence rebuilds once more
    assert sum(r for r, _ in S.capacity(calls, grow=False)) == S.CAP_BUILDS[-1] + 1
    # another order of the same geometries rebuilds; an empty group inserted does not
    more = S.capacity(calls + [[(1280, 720, 1), (640, 480, 1), (480, 640, 1)],
                               [(1280, 720, 1), (0, 0, 2), (640, 480, 1), (480, 640, 1)]])
    assert [r for r, _ in more[-2:]] == [True, False]


def test_frame_limit_groups():
    assert sum(B for _, _, B in S.LIMIT_GROUPS) == S.MAX_FRAMES
    for W, H, B in S.LIMIT_GROUPS:
        lay = S.Layout(*S.LIMIT_PARAMS[:3], W, H)
        assert lay.ok and lay.nftiles == 1 and lay.ncells == 1
