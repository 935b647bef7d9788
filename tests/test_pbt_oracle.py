"""CPU: the plain-Python restatement of one ``pbt`` call (oracle/pbt_oracle.py) against hand-worked populations — truncation
boundaries, goal and ties, explore on every parameter type at its bounds, resampling, failed trials and generation 0."""
import re

import numpy as np
import pytest

from oracle import pbt_oracle as O

L = O.LABEL
DNS_LABEL = re.compile(r"[a-z0-9]([-a-z0-9]{0,61}[a-z0-9])?")
SPACE = [{"name": "lr", "type": "double", "min": "0.1", "max": "1.0", "list": []},
         {"name": "layers", "type": "int", "min": "1", "max": "10", "list": []},
         {"name": "batch", "type": "discrete", "min": None, "max": None, "list": ["16", "32", "64"]},
         {"name": "opt", "type": "categorical", "min": None, "max": None, "list": ["sgd", "adam", "ftrl"]}]
PARAMS = {"lr": "0.5", "layers": "5", "batch": "32", "opt": "adam"}


class Script:
    """Scripted uniforms first, then a seeded Generator's (the trial names)."""

    def __init__(self, *us):
        self.us, self.rest = list(us), np.random.default_rng(0)

    @staticmethod
    def names(n):
        """Uniforms for n distinct trial names (trial j spells its j-th letter 8 times)."""
        return [(j + 0.5) / 36 for j in range(n) for _ in range(8)]

    def random(self):
        return self.us.pop(0) if self.us else float(self.rest.random())


def trial(name, objective=None, condition="succeeded", generation=0, parent=None, predecessor=None, params=None):
    return dict(name=name, objective=objective, condition=condition, generation=generation, parent=parent, predecessor=predecessor,
                params=dict(params or PARAMS))


def settings(n, threshold=0.2, resample=None):
    return {"n_population": n, "truncation_threshold": threshold, "resample_probability": resample}


def by_predecessor(out):
    return {o["labels"].get(L + "predecessor"): o for o in out}


@pytest.mark.parametrize("n,threshold,cut", [(5, 0.2, 1), (6, 0.2, 1), (40, 0.2, 8), (41, 0.2, 8),
                                             (5, 0.5, 2), (6, 0.5, 3), (40, 0.5, 20), (41, 0.5, 20)])
def test_truncation_boundaries(n, threshold, cut):
    assert O.truncation_count(threshold, n) == cut
    pop = [trial(f"m{i:02d}", objective=float(i)) for i in range(n)]         # MINIMIZE: m00 is the best, m{n-1} the worst
    out = O.step(pop, SPACE, "MINIMIZE", settings(n, threshold), np.random.default_rng(1), n, "exp")
    assert len(out) == n
    got = by_predecessor(out)
    for i in range(n):
        o = got[f"m{i:02d}"]
        if i >= n - cut:                                                      # bottom: a child of a top member
            assert int(o["copy_from"][1:]) < cut and o["labels"][L + "parent"] == o["copy_from"]
        else:                                                                 # the rest continue their own lineage
            assert o["copy_from"] == f"m{i:02d}" and o["params"] == PARAMS
        assert o["labels"][L + "generation"] == "1"


def test_parent_pick_is_uniform_over_the_top():
    pop = [trial(f"m{i:02d}", objective=float(i)) for i in range(10)]        # cut = 2 at 0.2: top m00, m01; bottom m08, m09
    for u, parent in ((0.0, "m00"), (0.4999, "m00"), (0.5, "m01"), (0.9999, "m01")):
        # served in (generation, name) order: m00..m07 continue (no draws), m08 draws u, then 4 explore uniforms, then a name
        out = O.step(pop, SPACE, "MINIMIZE", settings(10), Script(*Script.names(8), u), 10, "exp")
        assert by_predecessor(out)["m08"]["copy_from"] == parent


@pytest.mark.parametrize("goal,worst,best", [("MINIMIZE", "d", "b"), ("MAXIMIZE", "b", "d")])
def test_goal_decides_the_order(goal, worst, best):
    pop = [trial(n, objective=y) for n, y in zip("abcde", (3.0, 1.0, 2.0, 5.0, 4.0))]
    got = by_predecessor(O.step(pop, SPACE, goal, settings(5), np.random.default_rng(2), 5, "exp"))
    assert got[worst]["copy_from"] == best
    assert all(got[n]["copy_from"] == n for n in "abcde" if n != worst)


def test_ties_go_to_the_lower_generation_then_the_name():
    gens = {"a": 0, "b": 2, "c": 1, "d": 2, "e": 0}
    pop = [trial(n, objective=1.0, generation=g) for n, g in gens.items()]
    assert [t["name"] for t in O.rank_members(pop, "MINIMIZE")] == ["a", "e", "c", "b", "d"]
    assert [t["name"] for t in O.rank_members(pop, "MAXIMIZE")] == ["a", "e", "c", "b", "d"]
    got = by_predecessor(O.step(pop, SPACE, "MINIMIZE", settings(5), np.random.default_rng(3), 5, "exp"))
    assert got["d"]["copy_from"] == "a" and got["d"]["labels"][L + "generation"] == "1"
    assert got["b"]["copy_from"] == "b" and got["b"]["labels"][L + "generation"] == "3"


@pytest.mark.parametrize("value,u,expect", [("0.5", 0.1, repr(0.5 * 0.8)), ("0.5", 0.9, repr(0.5 * 1.2)),
                                            ("1.0", 0.9, "1.0"), ("0.9", 0.5, "1.0"), ("0.1", 0.2, "0.1"), ("0.12", 0.2, "0.1")])
def test_explore_double_clips(value, u, expect):
    assert O.perturb(SPACE[0], value, u) == expect


@pytest.mark.parametrize("lo,hi,value,u,expect", [
    (1, 10, "5", 0.9, "6"), (1, 10, "5", 0.1, "4"),
    (1, 10, "10", 0.9, "10"),                   # 12 clipped
    (1, 10, "9", 0.9, "10"),                    # 10.8 → 11, clipped
    (1, 10, "1", 0.1, "1"),                     # 0.8 rounds back to 1, steps down to 0, clipped
    (1, 10, "1", 0.9, "2"),                     # 1.2 rounds back to 1, steps up
    (1, 10, "2", 0.1, "1"), (1, 10, "2", 0.9, "3"),
    (-5, 5, "0", 0.9, "1"), (-5, 5, "0", 0.1, "-1"),
    (-5, 5, "-2", 0.9, "-3"), (-5, 5, "-2", 0.1, "-1"),
    (-5, 5, "-5", 0.9, "-5"), (-5, 5, "5", 0.9, "5"),
])
def test_explore_int_rounds_steps_and_clips(lo, hi, value, u, expect):
    spec = {"name": "k", "type": "int", "min": str(lo), "max": str(hi), "list": []}
    assert O.perturb(spec, value, u) == expect


@pytest.mark.parametrize("spec", SPACE[2:], ids=["discrete", "categorical"])
def test_explore_lists_move_to_a_neighbour_clamped_at_the_ends(spec):
    lst = spec["list"]
    assert O.perturb(spec, lst[0], 0.1) == lst[0] and O.perturb(spec, lst[0], 0.9) == lst[1]
    assert O.perturb(spec, lst[1], 0.1) == lst[0] and O.perturb(spec, lst[1], 0.9) == lst[2]
    assert O.perturb(spec, lst[-1], 0.9) == lst[-1] and O.perturb(spec, lst[-1], 0.1) == lst[-2]


def test_prior_draws():
    assert O.prior_draw(SPACE[0], 0.0) == "0.1" and O.prior_draw(SPACE[0], 0.5) == repr(0.1 + 0.5 * (1.0 - 0.1))
    assert O.prior_draw(SPACE[1], 0.0) == "1" and O.prior_draw(SPACE[1], 0.0999) == "1" and O.prior_draw(SPACE[1], 0.1) == "2"
    assert O.prior_draw(SPACE[1], 0.99999) == "10"
    assert [O.prior_draw(SPACE[3], u) for u in (0.0, 0.34, 0.67, 0.999)] == ["sgd", "adam", "ftrl", "ftrl"]


def _exploited(resample, script):
    pop = [trial(f"m{i}", objective=float(i)) for i in range(5)]              # cut = 1: m4 copies m0
    out = O.step(pop, SPACE, "MINIMIZE", settings(5, resample=resample), Script(*Script.names(4), *script), 5, "exp")
    o = by_predecessor(out)["m4"]
    assert o["copy_from"] == "m0"
    return o["params"]


def test_resample_probability_one_redraws_every_parameter():
    us = [0.3, 0.999, 0.2, 0.25, 0.1, 0.5, 0.0, 0.7]                         # (test, draw) per parameter
    assert _exploited(1.0, [0.0, *us]) == {"lr": repr(0.1 + 0.999 * (1.0 - 0.1)), "layers": "3", "batch": "32", "opt": "ftrl"}


def test_resample_probability_zero_always_perturbs():
    us = [0.999, 0.9, 0.999, 0.1, 0.999, 0.9, 0.999, 0.1]
    assert _exploited(0.0, [0.0, *us]) == {"lr": repr(0.5 * 1.2), "layers": "4", "batch": "64", "opt": "sgd"}


def test_without_resample_probability_no_test_draw_is_taken():
    assert _exploited(None, [0.0, 0.9, 0.1, 0.9, 0.1]) == {"lr": repr(0.5 * 1.2), "layers": "4", "batch": "64", "opt": "sgd"}


def test_failed_and_metricless_trials_end_their_lineage():
    pop = [trial("a", objective=1.0), trial("b", objective=2.0),
           trial("c", condition="failed", generation=3, parent="x", predecessor="x"),
           trial("d", objective=None, generation=2, parent="y", predecessor="y"),               # succeeded without a metric
           trial("e", condition="running", generation=1, parent="a0", predecessor="a0"),       # member: its predecessor
           trial("a0", objective=9.0), trial("x", objective=0.5), trial("y", objective=0.6),
           trial("f", condition="running", predecessor="z"), trial("z", condition="failed")]  # a fresh start: no member
    out = O.step(pop, SPACE, "MINIMIZE", settings(6), np.random.default_rng(4), 10, "exp")
    got = by_predecessor(out)
    assert set(got) == {"a", "b", "c", "d"}                                   # e and f are running; x, y, a0, z are superseded
    for n in ("c", "d"):
        assert got[n]["copy_from"] is None and L + "parent" not in got[n]["labels"] and got[n]["labels"][L + "generation"] == "0"
    # members a (1.0), b (2.0), a0 (9.0): cut = 0 at 0.2 × 3, so a and b continue
    assert got["a"]["copy_from"] == "a" and got["b"]["copy_from"] == "b"
    assert [o["labels"][L + "predecessor"] for o in out] == ["a", "b", "d", "c"]   # lowest generation first, then name


def test_generation_zero_fills_the_population_first():
    out = O.step([], SPACE, "MINIMIZE", settings(5), np.random.default_rng(5), 3, "exp")
    assert len(out) == 3 and all(o["labels"] == {L + "generation": "0"} and o["copy_from"] is None for o in out)
    pop = [trial(o["trial_name"], condition="running", params=o["params"]) for o in out]
    pop[0]["condition"], pop[0]["objective"] = "succeeded", 1.0
    more = O.step(pop, SPACE, "MINIMIZE", settings(5), np.random.default_rng(6), 10, "exp")
    assert len(more) == 3 and [o["copy_from"] for o in more] == [None, None, pop[0]["name"]]


@pytest.mark.parametrize("experiment,prefix", [("exp", "exp-"), ("A" * 80, "a" * 54 + "-"), ("../x", "x-"), ("..", ""),
                                               ("My_Exp.v2", "my-exp-v2-")])
def test_trial_names_are_dns_labels(experiment, prefix):
    out = O.step([], SPACE, "MINIMIZE", settings(5), np.random.default_rng(7), 5, experiment)
    for o in out:
        assert o["trial_name"].startswith(prefix) and len(o["trial_name"]) == len(prefix) + 8
        assert len(o["trial_name"]) <= 63 and DNS_LABEL.fullmatch(o["trial_name"])
    assert len({o["trial_name"] for o in out}) == 5
